// rbk_napi.cc — thin Node N-API addon over include/rbk_knn.h (librbk_knn.so).
//
// The build image has no node and no node_api.h: this is the binding a RunbookAI maintainer adds
// next to better-sqlite3.  It has never met real Node; it IS compiled (-Wall -Wextra -Werror), linked
// against librbk_knn.so and run in the test suite against a mock of the N-API subset it uses
// (napi/mock/, tests/test_napi_addon.py: every method, the promise / async-work path, every error
// path, results bit-identical to the oracle on an H100).  Logic-free by design: every method
// maps 1:1 onto a C-ABI call; errors become `new Error(rbk_last_error())` (sync methods
// throw, `search` rejects its Promise), the convention the reference already follows
// (vector-store.ts:197-199, embedder.ts:169-171).
//
//   const { RbkIndex } = require('./build/Release/rbk_knn.node')
//   const ix = new RbkIndex(dim, device, capacityHint)          // one GPU  (rbk_index_*)
//   const ix = new RbkIndex(dim, [0, 1, 2, 3], capacityHint)    // several GPUs behind one handle (rbk_group_*)
//   const ix = new RbkIndex(dim, device, capacityHint, hostRows) // hostRows != 0: exact rows in pinned host RAM
//   const ix = new RbkIndex(dim, device, capacityHint, hostRows, scanF16, exactRows)   // exactRows 'f64' | 'f32' | 'f32_split'
//                                              // (absent: RUNBOOK_KNN_EXACT_ROWS, else 'f64')
//   ix.appendF64(Float64Array rows)            -> firstSlot
//   ix.appendBlobs(Buffer[] blobs)             -> firstSlot     // SQLite f64-LE BLOBs, packed in C++: no JS copies
//   ix.overwriteF64(slot, Float64Array row); ix.overwriteF64Batch(BigInt64Array slots, Float64Array rows)
//   ix.tombstone(BigInt64Array slots); ix.clear()
//   ix.compact()                               -> BigInt64Array oldToNew   // reclaim tombstoned slots
//   ix.trim()                                  // give unused device memory back (after compact / clear)
//   ix.setTier({ f64OnHost, scanF16, exactRows })   // move the exact rows / switch the scan / widen or narrow them in
//                                              // place (omitted: kept)
//   ix.tier                                    -> { f64OnHost: boolean, scanF16: boolean, exactRows: 'f64' | 'f32' | 'f32_split' }
//   With exactRows 'f32' or 'f32_split', an append or overwrite holding a value no float32 can hold (RBK_ENOTF32,
//   nothing written)
//   widens the index to 'f64' in place and is repeated once, so the addon accepts every embedding a default index does.
//   await ix.search(Float64Array queries, B, kFetch, minScore)
//        -> { slots: BigInt64Array, scores: Float64Array, counts: Int32Array }
//   await ix.searchLarge(Float64Array queries, B, kFetch, minScore)   // kFetch up to 4096, same result object
//   await ix.searchUnbounded(Float64Array queries, B, kFetch, minScore)   // any kFetch >= 1, same result object
//   await ix.searchEach(Float64Array queries, B, Int32Array kFetch, Float64Array minScore)   // each query at its own
//        kFetch[b] and minScore[b]: the same result object with rows of K = max(kFetch) entries
//   ix.hasSearchEach                           -> boolean: the library has searchEach (else it throws)
//   await ix.searchSlots(BigInt64Array slots, B, Int32Array kFetch, Float64Array minScore)   // searchEach whose
//        queries are the stored rows of those global slots, read where the index keeps them: the same result object
//   ix.hasSearchSlots                          -> boolean: the library has searchSlots (else it throws)
//   await ix.searchMmr(Float64Array queries, B, Int32Array k, Int32Array fetchK, Float64Array lambdaMult,
//                      Float64Array minScore)   // diverse hits by maximal marginal relevance: query b's k[b] picks
//        from its fetchK[b] best, in selection order with their relevance: the result object with rows of max(k)
//   ix.hasSearchMmr                            -> boolean: the library has searchMmr (else it throws)
//   await ix.similarPairs(minScore, firstSlot, maxPairs)   // one page of every pair of live slots a < b with cosine
//        >= minScore, rows a from firstSlot on, at most maxPairs (>= size()) entries, whole rows only
//        -> { a: BigInt64Array, b: BigInt64Array, scores: Float64Array, nextSlot }   // nextSlot == size(): done
//   ix.hasSimilarPairs                         -> boolean: the library has similarPairs (else it throws)
//
// Build (where Node headers exist):  node-gyp with  libraries: ["-lrbk_knn"], include_dirs: ["../include"].
#include <node_api.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../include/rbk_knn.h"

// The large-k entry points came after ABI version 2 was fixed, so a librbk_knn.so of the same version may lack them.
// Weak references keep the addon loadable against such a library; `searchLarge` then throws instead of the module
// failing to load.
#pragma weak rbk_index_search_large_f64
#pragma weak rbk_group_search_large_f64
// The same for the unbounded search; `searchUnbounded` throws where it is missing.
#pragma weak rbk_index_search_unbounded_f64
#pragma weak rbk_group_search_unbounded_f64
// The same for compaction; `compact` throws where it is missing.  rbk_index_size, which sizes the map, is weak with it
// so that the method as a whole needs nothing a library without compaction may lack.
#pragma weak rbk_index_compact
#pragma weak rbk_index_size
// Compaction of a device group came later still; `compact` on a group handle throws where it is missing.
// rbk_group_size sizes its map.
#pragma weak rbk_group_compact
#pragma weak rbk_group_size
// The same for trim; `trim` throws where it is missing.
#pragma weak rbk_index_trim
#pragma weak rbk_group_trim
// The same for tier changes; `setTier` and `tier` throw where they are missing.
#pragma weak rbk_index_flags
#pragma weak rbk_index_set_tier
#pragma weak rbk_group_set_tier
#pragma weak rbk_group_member
// The same for the per-query search; `searchEach` throws where it is missing.
#pragma weak rbk_index_search_each_f64
#pragma weak rbk_group_search_each_f64
// The same for stored rows as queries; `searchSlots` throws where it is missing.
#pragma weak rbk_index_search_slots_f64
#pragma weak rbk_group_search_slots_f64
// The same for diverse hits by maximal marginal relevance; `searchMmr` throws where it is missing.
#pragma weak rbk_index_search_mmr_f64
#pragma weak rbk_group_search_mmr_f64
// The same for every pair above a threshold; `similarPairs` throws where it is missing.
#pragma weak rbk_index_similar_pairs_f64
#pragma weak rbk_group_similar_pairs_f64

namespace {

#define NAPI_OK(call)                                        \
  if ((call) != napi_ok) {                                   \
    napi_throw_error(env, nullptr, "N-API call failed: " #call); \
    return nullptr;                                          \
  }

napi_value throw_rbk(napi_env env) {
  napi_throw_error(env, nullptr, rbk_last_error());
  return nullptr;
}

// One JS object = one rbk_index (a device ordinal was given) or one rbk_group (an array of ordinals): the two
// families of the C ABI have the same shape, so every method below is a two-way switch and nothing else.
struct Handle {
  rbk_index* ix = nullptr;
  rbk_group* grp = nullptr;
  int32_t dim = 0;
  // A float32-row index refuses a value no float32 holds (RBK_ENOTF32) before writing anything: widen it to float64
  // rows in place and repeat the call once.
  template <typename F>
  rbk_status widening(F&& call) {
    rbk_status st = call();
    if (st != RBK_ENOTF32 || !has_tier()) return st;
    if ((st = set_tier((flags() & ~(RBK_INDEX_KEEP_F32 | RBK_INDEX_KEEP_F32_SPLIT)) | RBK_INDEX_KEEP_F64)) != RBK_OK)
      return st;
    return call();
  }
  rbk_status append_f64(const double* rows, int64_t n, int64_t* first) {
    return widening([&] {
      return grp ? rbk_group_append_f64(grp, rows, n, first) : rbk_index_append_f64(ix, rows, n, first);
    });
  }
  rbk_status overwrite_batch(const int64_t* slots, int64_t n, const double* rows) {
    return widening([&] {
      return grp ? rbk_group_overwrite_f64_batch(grp, slots, n, rows)
                 : rbk_index_overwrite_f64_batch(ix, slots, n, rows);
    });
  }
  rbk_status tombstone(const int64_t* slots, int64_t n) {
    return grp ? rbk_group_tombstone(grp, slots, n) : rbk_index_tombstone(ix, slots, n);
  }
  rbk_status clear() { return grp ? rbk_group_clear(grp) : rbk_index_clear(ix); }
  bool has_trim() const { return grp ? rbk_group_trim != nullptr : rbk_index_trim != nullptr; }
  rbk_status trim() { return grp ? rbk_group_trim(grp) : rbk_index_trim(ix); }
  int64_t count() const { return grp ? rbk_group_count(grp) : rbk_index_count(ix); }
  bool has_tier() const {
    return rbk_index_flags != nullptr &&
           (grp ? rbk_group_set_tier != nullptr && rbk_group_member != nullptr : rbk_index_set_tier != nullptr);
  }
  uint32_t flags() { return rbk_index_flags(grp ? rbk_group_member(grp, 0) : ix); }   // a group's members share them
  rbk_status set_tier(uint32_t flags) { return grp ? rbk_group_set_tier(grp, flags) : rbk_index_set_tier(ix, flags); }
  rbk_status search(const double* q, int32_t B, int32_t qdim, int32_t k, double ms, int64_t* s, double* v, int32_t* c) {
    return grp ? rbk_group_search_f64(grp, q, B, qdim, k, ms, s, v, c, nullptr)
               : rbk_index_search_f64(ix, q, B, qdim, k, ms, s, v, c, nullptr);
  }
  bool has_search_large() const {
    return grp ? rbk_group_search_large_f64 != nullptr : rbk_index_search_large_f64 != nullptr;
  }
  rbk_status search_large(const double* q, int32_t B, int32_t qdim, int32_t k, double ms, int64_t* s, double* v,
                          int32_t* c) {
    return grp ? rbk_group_search_large_f64(grp, q, B, qdim, k, ms, s, v, c, nullptr)
               : rbk_index_search_large_f64(ix, q, B, qdim, k, ms, s, v, c, nullptr);
  }
  bool has_search_unbounded() const {
    return grp ? rbk_group_search_unbounded_f64 != nullptr : rbk_index_search_unbounded_f64 != nullptr;
  }
  rbk_status search_unbounded(const double* q, int32_t B, int32_t qdim, int32_t k, double ms, int64_t* s, double* v,
                              int32_t* c) {
    return grp ? rbk_group_search_unbounded_f64(grp, q, B, qdim, k, ms, s, v, c, nullptr)
               : rbk_index_search_unbounded_f64(ix, q, B, qdim, k, ms, s, v, c, nullptr);
  }
  bool has_search_each() const {
    return grp ? rbk_group_search_each_f64 != nullptr : rbk_index_search_each_f64 != nullptr;
  }
  rbk_status search_each(const double* q, int32_t B, int32_t qdim, const int32_t* k, const double* ms, int64_t* s,
                         double* v, int32_t* c) {
    return grp ? rbk_group_search_each_f64(grp, q, B, qdim, k, ms, s, v, c, nullptr)
               : rbk_index_search_each_f64(ix, q, B, qdim, k, ms, s, v, c, nullptr);
  }
  bool has_search_slots() const {
    return grp ? rbk_group_search_slots_f64 != nullptr : rbk_index_search_slots_f64 != nullptr;
  }
  rbk_status search_slots(const int64_t* q, int32_t B, const int32_t* k, const double* ms, int64_t* s, double* v,
                          int32_t* c) {
    return grp ? rbk_group_search_slots_f64(grp, q, B, k, ms, s, v, c, nullptr)
               : rbk_index_search_slots_f64(ix, q, B, k, ms, s, v, c, nullptr);
  }
  bool has_search_mmr() const {
    return grp ? rbk_group_search_mmr_f64 != nullptr : rbk_index_search_mmr_f64 != nullptr;
  }
  rbk_status search_mmr(const double* q, int32_t B, int32_t qdim, const int32_t* k, const int32_t* f, const double* l,
                        const double* ms, int64_t* s, double* v, int32_t* c) {
    return grp ? rbk_group_search_mmr_f64(grp, q, B, qdim, k, f, l, ms, s, v, c, nullptr)
               : rbk_index_search_mmr_f64(ix, q, B, qdim, k, f, l, ms, s, v, c, nullptr);
  }
  bool has_similar_pairs() const {
    return grp ? rbk_group_similar_pairs_f64 != nullptr : rbk_index_similar_pairs_f64 != nullptr;
  }
  rbk_status similar_pairs(double ms, int64_t first, int64_t max_pairs, int64_t* a, int64_t* b, double* v, int64_t* n,
                           int64_t* next) {
    return grp ? rbk_group_similar_pairs_f64(grp, ms, first, max_pairs, a, b, v, n, next, nullptr)
               : rbk_index_similar_pairs_f64(ix, ms, first, max_pairs, a, b, v, n, next, nullptr);
  }
};

Handle* unwrap(napi_env env, napi_callback_info info, size_t* argc, napi_value* argv) {
  napi_value self;
  void* p = nullptr;
  if (napi_get_cb_info(env, info, argc, argv, &self, nullptr) != napi_ok) return nullptr;
  if (napi_unwrap(env, self, &p) != napi_ok) return nullptr;
  return static_cast<Handle*>(p);
}

void finalize_index(napi_env, void* data, void*) {
  Handle* h = static_cast<Handle*>(data);
  if (h->grp) rbk_group_destroy(h->grp);
  else rbk_index_destroy(h->ix);
  delete h;
}

// 'f64' / 'f32' / 'f32_split' -> the keep bit; anything else -> 0.
uint32_t keep_bit(const std::string& s) {
  return s == "f64" ? RBK_INDEX_KEEP_F64
                    : (s == "f32" ? RBK_INDEX_KEEP_F32 : (s == "f32_split" ? RBK_INDEX_KEEP_F32_SPLIT : 0u));
}

// A JS string (at most 15 bytes are needed here); false if v is not a string.
bool get_string(napi_env env, napi_value v, std::string* out) {
  char buf[16];
  size_t n = 0;
  if (napi_get_value_string_utf8(env, v, buf, sizeof buf, &n) != napi_ok) return false;
  out->assign(buf, n);
  return true;
}

napi_value New(napi_env env, napi_callback_info info) {
  size_t argc = 6;
  napi_value argv[6], self;
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, &self, nullptr));
  int32_t dim = 0, device = 0, host_rows = 0, scan_f16 = 0;
  int64_t hint = 0;
  NAPI_OK(napi_get_value_int32(env, argv[0], &dim));
  if (argc > 2) napi_get_value_int64(env, argv[2], &hint);
  if (argc > 3) napi_get_value_int32(env, argv[3], &host_rows);
  if (argc > 4) napi_get_value_int32(env, argv[4], &scan_f16);
  // exactRows (RUNBOOK_KNN_EXACT_ROWS when absent): 'f64' keeps the exact rows as float64, 'f32' as float32,
  // 'f32_split' as float32 split into the scan copy and low halves (the refusal names the two plain widths)
  std::string exact_rows;
  if (argc > 5) {
    if (!get_string(env, argv[5], &exact_rows)) exact_rows = "?";
  } else {
    const char* e = getenv("RUNBOOK_KNN_EXACT_ROWS");
    exact_rows = e && *e ? e : "f64";
  }
  const uint32_t keep = keep_bit(exact_rows);
  if (keep == 0) {
    napi_throw_type_error(env, nullptr, "exactRows must be 'f64' or 'f32'");
    return nullptr;
  }
  Handle* h = new Handle();
  h->dim = dim;
  bool is_array = false;
  if (argc > 1) napi_is_array(env, argv[1], &is_array);
  // KEEP_F64: the reference stores float64 embeddings; keep them so results are exact for any input (KEEP_F32: the
  // same answers from float32 rows while every value is a float32).  hostRows (RUNBOOK_KNN_F64_ON_HOST in
  // ts/gpu-embedding-index.ts): keep them in pinned host memory instead of on the GPU.  scanF16
  // (RUNBOOK_KNN_SCAN_F16): the scan reads per-row scaled fp16 rows instead of bf16 (same answers).
  const uint32_t flags = keep | (host_rows != 0 ? RBK_INDEX_F64_ON_HOST : 0u) |
                         (scan_f16 != 0 ? RBK_INDEX_SCAN_F16 : 0u);
  rbk_status st;
  if (is_array) {   // [0, 1, ...]: the corpus sharded over these GPUs, one call per search (rbk_group_*)
    uint32_t n = 0;
    napi_get_array_length(env, argv[1], &n);
    std::vector<int32_t> devs(n);
    for (uint32_t i = 0; i < n; ++i) {
      napi_value e;
      napi_get_element(env, argv[1], i, &e);
      napi_get_value_int32(env, e, &devs[i]);
    }
    st = rbk_group_create(dim, devs.data(), (int32_t)n, hint, flags, &h->grp);
  } else {
    if (argc > 1) napi_get_value_int32(env, argv[1], &device);
    st = rbk_index_create_ex(dim, device, hint, flags, &h->ix);
  }
  if (st != RBK_OK) {
    delete h;
    return throw_rbk(env);   // no GPU -> throws, no fallback
  }
  NAPI_OK(napi_wrap(env, self, h, finalize_index, nullptr, nullptr));
  return self;
}

napi_value AppendF64(napi_env env, napi_callback_info info) {
  size_t argc = 1;
  napi_value argv[1];
  Handle* h = unwrap(env, info, &argc, argv);
  napi_typedarray_type t;
  size_t len;
  void* data;
  NAPI_OK(napi_get_typedarray_info(env, argv[0], &t, &len, &data, nullptr, nullptr));
  if (t != napi_float64_array || len % h->dim != 0) {
    napi_throw_error(env, nullptr, "Vectors must have the same length");
    return nullptr;
  }
  int64_t first = -1;
  if (h->append_f64(static_cast<const double*>(data), (int64_t)(len / h->dim), &first) != RBK_OK) return throw_rbk(env);
  napi_value out;
  NAPI_OK(napi_create_int64(env, first, &out));
  return out;
}

// appendBlobs(Buffer[]): the `embedding` BLOBs exactly as better-sqlite3 returns them (float64 LE, 8*dim bytes
// each, vector-store.ts:71-88).  Packed with memcpy here and handed over in one call: no per-row JS work at all.
napi_value AppendBlobs(napi_env env, napi_callback_info info) {
  size_t argc = 1;
  napi_value argv[1];
  Handle* h = unwrap(env, info, &argc, argv);
  uint32_t n = 0;
  NAPI_OK(napi_get_array_length(env, argv[0], &n));
  std::vector<double> packed((size_t)n * h->dim);
  for (uint32_t i = 0; i < n; ++i) {
    napi_value e;
    void* data;
    size_t len;
    NAPI_OK(napi_get_element(env, argv[0], i, &e));
    NAPI_OK(napi_get_buffer_info(env, e, &data, &len));
    if (len != (size_t)h->dim * 8) {
      napi_throw_error(env, nullptr, "Vectors must have the same length");
      return nullptr;
    }
    memcpy(&packed[(size_t)i * h->dim], data, len);
  }
  int64_t first = -1;
  if (h->append_f64(packed.data(), n, &first) != RBK_OK) return throw_rbk(env);
  napi_value out;
  NAPI_OK(napi_create_int64(env, first, &out));
  return out;
}

napi_value OverwriteF64(napi_env env, napi_callback_info info) {
  size_t argc = 2;
  napi_value argv[2];
  Handle* h = unwrap(env, info, &argc, argv);
  int64_t slot;
  NAPI_OK(napi_get_value_int64(env, argv[0], &slot));
  napi_typedarray_type t;
  size_t len;
  void* data;
  NAPI_OK(napi_get_typedarray_info(env, argv[1], &t, &len, &data, nullptr, nullptr));
  if (t != napi_float64_array || (int32_t)len != h->dim) {
    napi_throw_error(env, nullptr, "Vectors must have the same length");
    return nullptr;
  }
  if (h->overwrite_batch(&slot, 1, static_cast<const double*>(data)) != RBK_OK) return throw_rbk(env);
  return nullptr;
}

// overwriteF64Batch(BigInt64Array slots, Float64Array rows): addChunks over ids that already exist - one call,
// one host round trip for the whole document.
napi_value OverwriteF64Batch(napi_env env, napi_callback_info info) {
  size_t argc = 2;
  napi_value argv[2];
  Handle* h = unwrap(env, info, &argc, argv);
  napi_typedarray_type ts, tr;
  size_t ns, nr;
  void *ds, *dr;
  NAPI_OK(napi_get_typedarray_info(env, argv[0], &ts, &ns, &ds, nullptr, nullptr));
  NAPI_OK(napi_get_typedarray_info(env, argv[1], &tr, &nr, &dr, nullptr, nullptr));
  if (ts != napi_bigint64_array || tr != napi_float64_array || nr != ns * (size_t)h->dim) {
    napi_throw_error(env, nullptr, "Vectors must have the same length");
    return nullptr;
  }
  if (h->overwrite_batch(static_cast<const int64_t*>(ds), (int64_t)ns, static_cast<const double*>(dr)) != RBK_OK)
    return throw_rbk(env);
  return nullptr;
}

napi_value Tombstone(napi_env env, napi_callback_info info) {
  size_t argc = 1;
  napi_value argv[1];
  Handle* h = unwrap(env, info, &argc, argv);
  napi_typedarray_type t;
  size_t len;
  void* data;
  NAPI_OK(napi_get_typedarray_info(env, argv[0], &t, &len, &data, nullptr, nullptr));
  if (t != napi_bigint64_array) {
    napi_throw_type_error(env, nullptr, "slots must be a BigInt64Array");
    return nullptr;
  }
  if (h->tombstone(static_cast<const int64_t*>(data), (int64_t)len) != RBK_OK) return throw_rbk(env);
  return nullptr;
}

napi_value Clear(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  if (h->clear() != RBK_OK) return throw_rbk(env);
  return nullptr;
}

// compact() -> BigInt64Array old_to_new: reclaim the slots of tombstoned rows; old slot s now lives at
// old_to_new[s] (-1 = it was deleted).  Synchronous.  On a device group the slots are global ones.
napi_value Compact(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  if (h->grp && (rbk_group_compact == nullptr || rbk_group_size == nullptr)) {
    napi_throw_error(env, nullptr, "compaction is not available for a device group");
    return nullptr;
  }
  if (!h->grp && (rbk_index_compact == nullptr || rbk_index_size == nullptr)) {
    napi_throw_error(env, nullptr, "compact: this librbk_knn.so has no compaction (rbk_index_compact)");
    return nullptr;
  }
  const int64_t n = h->grp ? rbk_group_size(h->grp) : rbk_index_size(h->ix);
  napi_value ab, out;
  void* p = nullptr;
  NAPI_OK(napi_create_arraybuffer(env, (size_t)n * 8, &p, &ab));
  int64_t* map = static_cast<int64_t*>(p);
  if ((h->grp ? rbk_group_compact(h->grp, map, n) : rbk_index_compact(h->ix, map, n)) != RBK_OK) return throw_rbk(env);
  NAPI_OK(napi_create_typedarray(env, napi_bigint64_array, (size_t)n, ab, 0, &out));
  return out;
}

// trim(): capacity down to what the rows need, scratch released; slots and answers unchanged.  Synchronous.
napi_value Trim(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  if (!h->has_trim()) {
    napi_throw_error(env, nullptr, "trim: this librbk_knn.so has no trim (rbk_index_trim / rbk_group_trim)");
    return nullptr;
  }
  if (h->trim() != RBK_OK) return throw_rbk(env);
  return nullptr;
}

bool require_tier(napi_env env, Handle* h) {
  if (h->has_tier()) return true;
  napi_throw_error(env, nullptr, "setTier: this librbk_knn.so has no tier change (rbk_index_set_tier / rbk_group_set_tier)");
  return false;
}

// setTier({ f64OnHost, scanF16, exactRows }): rbk_index_set_tier / rbk_group_set_tier.  A key that is absent keeps its
// setting; f64OnHost / scanF16 must be booleans, exactRows 'f64', 'f32' or 'f32_split'.  Synchronous; answers do not change.
napi_value SetTier(napi_env env, napi_callback_info info) {
  size_t argc = 1;
  napi_value argv[1] = {nullptr};
  Handle* h = unwrap(env, info, &argc, argv);
  if (!require_tier(env, h)) return nullptr;
  uint32_t flags = h->flags();
  const struct {
    const char* name;
    uint32_t bit;
  } keys[] = {{"f64OnHost", RBK_INDEX_F64_ON_HOST}, {"scanF16", RBK_INDEX_SCAN_F16}};
  for (const auto& k : keys) {
    bool has = false;
    if (argc < 1 || napi_has_named_property(env, argv[0], k.name, &has) != napi_ok) {
      napi_throw_type_error(env, nullptr, "setTier: the argument must be an object { f64OnHost, scanF16 }");
      return nullptr;
    }
    if (!has) continue;
    napi_value v;
    bool on = false;
    NAPI_OK(napi_get_named_property(env, argv[0], k.name, &v));
    if (napi_get_value_bool(env, v, &on) != napi_ok) {
      napi_throw_type_error(env, nullptr, (std::string("setTier: ") + k.name + " must be a boolean").c_str());
      return nullptr;
    }
    flags = on ? (flags | k.bit) : (flags & ~k.bit);
  }
  bool has = false;
  NAPI_OK(napi_has_named_property(env, argv[0], "exactRows", &has));
  if (has) {
    napi_value v;
    std::string s;
    NAPI_OK(napi_get_named_property(env, argv[0], "exactRows", &v));
    const uint32_t keep = get_string(env, v, &s) ? keep_bit(s) : 0u;
    if (keep == 0) {
      napi_throw_type_error(env, nullptr, "setTier: exactRows must be 'f64' or 'f32'");
      return nullptr;
    }
    flags = (flags & ~(RBK_INDEX_KEEP_F64 | RBK_INDEX_KEEP_F32 | RBK_INDEX_KEEP_F32_SPLIT)) | keep;
  }
  if (h->set_tier(flags) != RBK_OK) return throw_rbk(env);
  return nullptr;
}

// tier -> { f64OnHost, scanF16, exactRows }: where the exact rows live, which scan the index runs and the exact rows'
// width, as they are now.
napi_value GetTier(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  if (!require_tier(env, h)) return nullptr;
  const uint32_t flags = h->flags();
  napi_value out, host, f16;
  NAPI_OK(napi_create_object(env, &out));
  NAPI_OK(napi_get_boolean(env, (flags & RBK_INDEX_F64_ON_HOST) != 0, &host));
  NAPI_OK(napi_get_boolean(env, (flags & RBK_INDEX_SCAN_F16) != 0, &f16));
  NAPI_OK(napi_set_named_property(env, out, "f64OnHost", host));
  NAPI_OK(napi_set_named_property(env, out, "scanF16", f16));
  napi_value rows;
  const char* kept = (flags & RBK_INDEX_KEEP_F32) ? "f32" : ((flags & RBK_INDEX_KEEP_F32_SPLIT) ? "f32_split" : "f64");
  NAPI_OK(napi_create_string_utf8(env, kept, NAPI_AUTO_LENGTH, &rows));
  NAPI_OK(napi_set_named_property(env, out, "exactRows", rows));
  return out;
}

napi_value Count(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  napi_value out;
  NAPI_OK(napi_create_int64(env, h->count(), &out));
  return out;
}

// ---- search: runs on a libuv worker so the JS thread never blocks on the GPU ----
// search / searchLarge / searchUnbounded / searchEach / searchSlots / searchMmr
enum class SearchKind { kScan, kLarge, kUnbounded, kEach, kSlots, kMmr };

struct SearchJob {
  Handle* ix;
  std::vector<double> queries;
  int32_t B, dim, k;
  SearchKind kind;
  double min_score;
  std::vector<int64_t> query_slots;  // searchSlots: the queries' global slots [B]
  std::vector<int32_t> k_each;      // searchEach, searchSlots: kFetch[B] and minScore[B]; k is then their largest k
  std::vector<double> min_each;
  std::vector<int32_t> fetch_each;   // searchMmr: fetchK[B] and lambdaMult[B]; k_each is then k[B], min_each minScore[B]
  std::vector<double> lambda_each;
  std::vector<int64_t> slots;
  std::vector<double> scores;
  std::vector<int32_t> counts;
  rbk_status st = RBK_OK;
  std::string err;
  napi_deferred deferred;
  napi_async_work work;
};

void search_execute(napi_env, void* data) {
  SearchJob* j = static_cast<SearchJob*>(data);
  if (j->kind == SearchKind::kSlots) {
    j->st = j->ix->search_slots(j->query_slots.data(), j->B, j->k_each.data(), j->min_each.data(), j->slots.data(),
                                j->scores.data(), j->counts.data());
    if (j->st != RBK_OK) j->err = rbk_last_error();
    return;
  }
  if (j->kind == SearchKind::kMmr) {
    j->st = j->ix->search_mmr(j->queries.data(), j->B, j->dim, j->k_each.data(), j->fetch_each.data(),
                              j->lambda_each.data(), j->min_each.data(), j->slots.data(), j->scores.data(),
                              j->counts.data());
    if (j->st != RBK_OK) j->err = rbk_last_error();
    return;
  }
  if (j->kind == SearchKind::kEach) {
    j->st = j->ix->search_each(j->queries.data(), j->B, j->dim, j->k_each.data(), j->min_each.data(), j->slots.data(),
                               j->scores.data(), j->counts.data());
    if (j->st != RBK_OK) j->err = rbk_last_error();
    return;
  }
  auto fn = j->kind == SearchKind::kLarge       ? &Handle::search_large
            : j->kind == SearchKind::kUnbounded ? &Handle::search_unbounded
                                                : &Handle::search;
  j->st = (j->ix->*fn)(j->queries.data(), j->B, j->dim, j->k, j->min_score, j->slots.data(), j->scores.data(),
                       j->counts.data());
  if (j->st != RBK_OK) j->err = rbk_last_error();   // thread-local: read it on the worker thread
}

void search_complete(napi_env env, napi_status, void* data) {
  SearchJob* j = static_cast<SearchJob*>(data);
  if (j->st != RBK_OK) {
    napi_value msg, error;
    napi_create_string_utf8(env, j->err.c_str(), NAPI_AUTO_LENGTH, &msg);
    napi_create_error(env, nullptr, msg, &error);
    napi_reject_deferred(env, j->deferred, error);
  } else {
    napi_value out, ab, ta;
    void* p;
    napi_create_object(env, &out);
    napi_create_arraybuffer(env, j->slots.size() * 8, &p, &ab);
    memcpy(p, j->slots.data(), j->slots.size() * 8);
    napi_create_typedarray(env, napi_bigint64_array, j->slots.size(), ab, 0, &ta);
    napi_set_named_property(env, out, "slots", ta);
    napi_create_arraybuffer(env, j->scores.size() * 8, &p, &ab);
    memcpy(p, j->scores.data(), j->scores.size() * 8);
    napi_create_typedarray(env, napi_float64_array, j->scores.size(), ab, 0, &ta);
    napi_set_named_property(env, out, "scores", ta);
    napi_create_arraybuffer(env, j->counts.size() * 4, &p, &ab);
    memcpy(p, j->counts.data(), j->counts.size() * 4);
    napi_create_typedarray(env, napi_int32_array, j->counts.size(), ab, 0, &ta);
    napi_set_named_property(env, out, "counts", ta);
    napi_resolve_deferred(env, j->deferred, out);
  }
  napi_delete_async_work(env, j->work);
  delete j;
}

napi_value QueueSearch(napi_env env, napi_callback_info info, SearchKind kind) {
  size_t argc = 4;
  napi_value argv[4];
  Handle* ix = unwrap(env, info, &argc, argv);
  if (kind == SearchKind::kLarge && !ix->has_search_large()) {
    napi_throw_error(env, nullptr, "searchLarge: this librbk_knn.so has no large-k search (rbk_*_search_large_f64)");
    return nullptr;
  }
  if (kind == SearchKind::kUnbounded && !ix->has_search_unbounded()) {
    napi_throw_error(env, nullptr,
                     "searchUnbounded: this librbk_knn.so has no unbounded search (rbk_*_search_unbounded_f64)");
    return nullptr;
  }
  if (kind == SearchKind::kEach && !ix->has_search_each()) {
    napi_throw_error(env, nullptr, "searchEach: this librbk_knn.so has no per-query search (rbk_*_search_each_f64)");
    return nullptr;
  }
  if (kind == SearchKind::kSlots && !ix->has_search_slots()) {
    napi_throw_error(env, nullptr, "searchSlots: this librbk_knn.so has no search by slot (rbk_*_search_slots_f64)");
    return nullptr;
  }
  const bool each = kind == SearchKind::kEach || kind == SearchKind::kSlots;
  const char* what = kind == SearchKind::kSlots ? "searchSlots" : "searchEach";
  napi_typedarray_type t;
  size_t len;
  void* data;
  NAPI_OK(napi_get_typedarray_info(env, argv[0], &t, &len, &data, nullptr, nullptr));
  if (kind == SearchKind::kSlots && t != napi_bigint64_array) {
    napi_throw_type_error(env, nullptr, "searchSlots: slots must be a BigInt64Array");
    return nullptr;
  }
  int32_t B = 0;
  napi_get_value_int32(env, argv[1], &B);
  std::vector<int32_t> k_each;
  std::vector<double> min_each;
  if (each) {   // kFetch: Int32Array[B], minScore: Float64Array[B] (-Infinity: no threshold)
    napi_typedarray_type tk, tm;
    size_t nk, nm;
    void *pk, *pm;
    if (napi_get_typedarray_info(env, argv[2], &tk, &nk, &pk, nullptr, nullptr) != napi_ok ||
        napi_get_typedarray_info(env, argv[3], &tm, &nm, &pm, nullptr, nullptr) != napi_ok ||
        tk != napi_int32_array || tm != napi_float64_array) {
      napi_throw_type_error(env, nullptr, (std::string(what) + ": kFetch must be an Int32Array and minScore a "
                                                          "Float64Array").c_str());
      return nullptr;
    }
    if (B < 0 || nk != static_cast<size_t>(B) || nm != static_cast<size_t>(B) ||
        (kind == SearchKind::kSlots && len != static_cast<size_t>(B))) {
      napi_throw_error(env, nullptr, (std::string(what) + ": kFetch and minScore need one entry per query").c_str());
      return nullptr;
    }
    k_each.assign(static_cast<int32_t*>(pk), static_cast<int32_t*>(pk) + nk);
    min_each.assign(static_cast<double*>(pm), static_cast<double*>(pm) + nm);
  }
  auto* j = new SearchJob();
  j->ix = ix;
  j->kind = kind;
  j->B = B;
  if (each) {
    // the row stride; a kFetch[b] < 1 leaves it at 0 or 1, and the library refuses the call with its own message
    j->k = 0;
    for (int32_t v : k_each) j->k = std::max(j->k, v);
    j->k_each = std::move(k_each);
    j->min_each = std::move(min_each);
  } else {
    napi_get_value_int32(env, argv[2], &j->k);
    napi_get_value_double(env, argv[3], &j->min_score);   // pass -Infinity for "no threshold"
  }
  if (kind == SearchKind::kSlots) {
    j->query_slots.assign(static_cast<int64_t*>(data), static_cast<int64_t*>(data) + len);
  } else {
    j->dim = j->B > 0 ? (int32_t)(len / (size_t)j->B) : 0;   // a wrong length surfaces as RBK_EDIM
    j->queries.assign(static_cast<double*>(data), static_cast<double*>(data) + len);
  }
  j->slots.resize((size_t)j->B * j->k);
  j->scores.resize((size_t)j->B * j->k);
  j->counts.resize((size_t)j->B);
  napi_value promise, name;
  NAPI_OK(napi_create_promise(env, &j->deferred, &promise));
  napi_create_string_utf8(env, "rbk_search", NAPI_AUTO_LENGTH, &name);
  NAPI_OK(napi_create_async_work(env, nullptr, name, search_execute, search_complete, j, &j->work));
  NAPI_OK(napi_queue_async_work(env, j->work));
  return promise;
}

napi_value Search(napi_env env, napi_callback_info info) { return QueueSearch(env, info, SearchKind::kScan); }
napi_value SearchLarge(napi_env env, napi_callback_info info) { return QueueSearch(env, info, SearchKind::kLarge); }
napi_value SearchUnbounded(napi_env env, napi_callback_info info) {
  return QueueSearch(env, info, SearchKind::kUnbounded);
}
napi_value SearchEach(napi_env env, napi_callback_info info) { return QueueSearch(env, info, SearchKind::kEach); }

napi_value SearchSlots(napi_env env, napi_callback_info info) { return QueueSearch(env, info, SearchKind::kSlots); }

// searchMmr(queries, B, k, fetchK, lambdaMult, minScore): one Int32Array or Float64Array entry per query each; the
// library checks the values, so a k[b] < 1 or a lambdaMult[b] outside [0, 1] rejects with its message.
napi_value SearchMmr(napi_env env, napi_callback_info info) {
  size_t argc = 6;
  napi_value argv[6];
  Handle* ix = unwrap(env, info, &argc, argv);
  if (!ix->has_search_mmr()) {
    napi_throw_error(env, nullptr, "searchMmr: this librbk_knn.so has no MMR search (rbk_*_search_mmr_f64)");
    return nullptr;
  }
  napi_typedarray_type t[6];
  size_t len[6] = {};
  void* data[6] = {};
  for (int i : {0, 2, 3, 4, 5}) {
    if (argc <= static_cast<size_t>(i) ||
        napi_get_typedarray_info(env, argv[i], &t[i], &len[i], &data[i], nullptr, nullptr) != napi_ok)
      t[i] = napi_uint8_array;   // not a typed array: refused below
  }
  if (t[0] != napi_float64_array || t[2] != napi_int32_array || t[3] != napi_int32_array ||
      t[4] != napi_float64_array || t[5] != napi_float64_array) {
    napi_throw_type_error(env, nullptr, "searchMmr: queries, lambdaMult and minScore must be Float64Arrays, k and "
                                        "fetchK Int32Arrays");
    return nullptr;
  }
  int32_t B = 0;
  napi_get_value_int32(env, argv[1], &B);
  if (B < 0 || len[2] != static_cast<size_t>(B) || len[3] != static_cast<size_t>(B) ||
      len[4] != static_cast<size_t>(B) || len[5] != static_cast<size_t>(B)) {
    napi_throw_error(env, nullptr, "searchMmr: k, fetchK, lambdaMult and minScore need one entry per query");
    return nullptr;
  }
  auto* j = new SearchJob();
  j->ix = ix;
  j->kind = SearchKind::kMmr;
  j->B = B;
  j->dim = B > 0 ? (int32_t)(len[0] / (size_t)B) : 0;   // a wrong length surfaces as RBK_EDIM
  j->queries.assign(static_cast<double*>(data[0]), static_cast<double*>(data[0]) + len[0]);
  j->k_each.assign(static_cast<int32_t*>(data[2]), static_cast<int32_t*>(data[2]) + B);
  j->fetch_each.assign(static_cast<int32_t*>(data[3]), static_cast<int32_t*>(data[3]) + B);
  j->lambda_each.assign(static_cast<double*>(data[4]), static_cast<double*>(data[4]) + B);
  j->min_each.assign(static_cast<double*>(data[5]), static_cast<double*>(data[5]) + B);
  j->k = 0;   // the row stride: the largest k (a k[b] < 1 is refused by the library)
  for (int32_t v : j->k_each) j->k = std::max(j->k, v);
  j->slots.resize((size_t)B * j->k);
  j->scores.resize((size_t)B * j->k);
  j->counts.resize((size_t)B);
  napi_value promise, name;
  NAPI_OK(napi_create_promise(env, &j->deferred, &promise));
  napi_create_string_utf8(env, "rbk_search_mmr", NAPI_AUTO_LENGTH, &name);
  NAPI_OK(napi_create_async_work(env, nullptr, name, search_execute, search_complete, j, &j->work));
  NAPI_OK(napi_queue_async_work(env, j->work));
  return promise;
}

napi_value HasSearchMmr(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  napi_value out;
  NAPI_OK(napi_get_boolean(env, h->has_search_mmr(), &out));
  return out;
}

napi_value HasSearchEach(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  napi_value out;
  NAPI_OK(napi_get_boolean(env, h->has_search_each(), &out));
  return out;
}

// ---- similarPairs: one page of the pairs, on a libuv worker like search ----
struct PairsJob {
  Handle* ix;
  double min_score;
  int64_t first, max_pairs, n = 0, next = 0;
  std::vector<int64_t> a, b;
  std::vector<double> scores;
  rbk_status st = RBK_OK;
  std::string err;
  napi_deferred deferred;
  napi_async_work work;
};

void pairs_execute(napi_env, void* data) {
  PairsJob* j = static_cast<PairsJob*>(data);
  j->st = j->ix->similar_pairs(j->min_score, j->first, j->max_pairs, j->a.data(), j->b.data(), j->scores.data(), &j->n,
                               &j->next);
  if (j->st != RBK_OK) j->err = rbk_last_error();
}

void pairs_complete(napi_env env, napi_status, void* data) {
  PairsJob* j = static_cast<PairsJob*>(data);
  if (j->st != RBK_OK) {
    napi_value msg, error;
    napi_create_string_utf8(env, j->err.c_str(), NAPI_AUTO_LENGTH, &msg);
    napi_create_error(env, nullptr, msg, &error);
    napi_reject_deferred(env, j->deferred, error);
  } else {
    napi_value out, ab, ta, next;
    void* p;
    const size_t n = static_cast<size_t>(j->n);
    napi_create_object(env, &out);
    napi_create_arraybuffer(env, n * 8, &p, &ab);
    memcpy(p, j->a.data(), n * 8);
    napi_create_typedarray(env, napi_bigint64_array, n, ab, 0, &ta);
    napi_set_named_property(env, out, "a", ta);
    napi_create_arraybuffer(env, n * 8, &p, &ab);
    memcpy(p, j->b.data(), n * 8);
    napi_create_typedarray(env, napi_bigint64_array, n, ab, 0, &ta);
    napi_set_named_property(env, out, "b", ta);
    napi_create_arraybuffer(env, n * 8, &p, &ab);
    memcpy(p, j->scores.data(), n * 8);
    napi_create_typedarray(env, napi_float64_array, n, ab, 0, &ta);
    napi_set_named_property(env, out, "scores", ta);
    napi_create_int64(env, j->next, &next);
    napi_set_named_property(env, out, "nextSlot", next);
    napi_resolve_deferred(env, j->deferred, out);
  }
  napi_delete_async_work(env, j->work);
  delete j;
}

napi_value SimilarPairs(napi_env env, napi_callback_info info) {
  size_t argc = 3;
  napi_value argv[3];
  Handle* ix = unwrap(env, info, &argc, argv);
  if (!ix->has_similar_pairs()) {
    napi_throw_error(env, nullptr, "similarPairs: this librbk_knn.so has no similar pairs (rbk_*_similar_pairs_f64)");
    return nullptr;
  }
  PairsJob* j = new PairsJob();
  j->ix = ix;
  napi_get_value_double(env, argv[0], &j->min_score);   // -Infinity: every pair
  napi_get_value_int64(env, argv[1], &j->first);
  napi_get_value_int64(env, argv[2], &j->max_pairs);
  // the library refuses a maxPairs below size() with its own message: the buffers are at least one entry (never null)
  // and never larger than asked
  const size_t cap = static_cast<size_t>(std::max<int64_t>(j->max_pairs, 1));
  try {
    j->a.resize(cap);
    j->b.resize(cap);
    j->scores.resize(cap);
  } catch (const std::exception&) {
    delete j;
    napi_throw_error(env, nullptr, "similarPairs: no host memory for maxPairs entries");
    return nullptr;
  }
  napi_value promise, name;
  NAPI_OK(napi_create_promise(env, &j->deferred, &promise));
  napi_create_string_utf8(env, "rbk_similar_pairs", NAPI_AUTO_LENGTH, &name);
  NAPI_OK(napi_create_async_work(env, nullptr, name, pairs_execute, pairs_complete, j, &j->work));
  NAPI_OK(napi_queue_async_work(env, j->work));
  return promise;
}

napi_value HasSimilarPairs(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  napi_value out;
  NAPI_OK(napi_get_boolean(env, h->has_similar_pairs(), &out));
  return out;
}

napi_value HasSearchSlots(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  napi_value out;
  NAPI_OK(napi_get_boolean(env, h->has_search_slots(), &out));
  return out;
}

napi_value Init(napi_env env, napi_value exports) {
  napi_property_descriptor props[] = {
      {"appendF64", nullptr, AppendF64, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"appendBlobs", nullptr, AppendBlobs, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"overwriteF64", nullptr, OverwriteF64, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"overwriteF64Batch", nullptr, OverwriteF64Batch, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"tombstone", nullptr, Tombstone, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"clear", nullptr, Clear, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"compact", nullptr, Compact, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"trim", nullptr, Trim, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"setTier", nullptr, SetTier, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"tier", nullptr, nullptr, GetTier, nullptr, nullptr, napi_default, nullptr},
      {"count", nullptr, Count, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"search", nullptr, Search, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"searchLarge", nullptr, SearchLarge, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"searchUnbounded", nullptr, SearchUnbounded, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"searchEach", nullptr, SearchEach, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"hasSearchEach", nullptr, nullptr, HasSearchEach, nullptr, nullptr, napi_default, nullptr},
      {"searchSlots", nullptr, SearchSlots, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"hasSearchSlots", nullptr, nullptr, HasSearchSlots, nullptr, nullptr, napi_default, nullptr},
      {"searchMmr", nullptr, SearchMmr, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"hasSearchMmr", nullptr, nullptr, HasSearchMmr, nullptr, nullptr, napi_default, nullptr},
      {"similarPairs", nullptr, SimilarPairs, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"hasSimilarPairs", nullptr, nullptr, HasSimilarPairs, nullptr, nullptr, napi_default, nullptr},
  };
  napi_value cls;
  NAPI_OK(napi_define_class(env, "RbkIndex", NAPI_AUTO_LENGTH, New, nullptr, sizeof props / sizeof props[0], props, &cls));
  NAPI_OK(napi_set_named_property(env, exports, "RbkIndex", cls));
  return exports;
}

}  // namespace

NAPI_MODULE(NODE_GYP_MODULE_NAME, Init)
