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
//   const ix = new RbkIndex(dim, device, capacityHint, hostRows) // hostRows != 0: float64 rows in pinned host RAM
//   ix.appendF64(Float64Array rows)            -> firstSlot
//   ix.appendBlobs(Buffer[] blobs)             -> firstSlot     // SQLite f64-LE BLOBs, packed in C++: no JS copies
//   ix.overwriteF64(slot, Float64Array row); ix.overwriteF64Batch(BigInt64Array slots, Float64Array rows)
//   ix.tombstone(BigInt64Array slots); ix.clear()
//   ix.compact()                               -> BigInt64Array oldToNew   // reclaim tombstoned slots (one GPU only)
//   ix.trim()                                  // give unused device memory back (after compact / clear)
//   await ix.search(Float64Array queries, B, kFetch, minScore)
//        -> { slots: BigInt64Array, scores: Float64Array, counts: Int32Array }
//   await ix.searchLarge(Float64Array queries, B, kFetch, minScore)   // kFetch up to 4096, same result object
//   await ix.searchUnbounded(Float64Array queries, B, kFetch, minScore)   // any kFetch >= 1, same result object
//
// Build (where Node headers exist):  node-gyp with  libraries: ["-lrbk_knn"], include_dirs: ["../include"].
#include <node_api.h>

#include <cmath>
#include <cstdint>
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
// The same for trim; `trim` throws where it is missing.
#pragma weak rbk_index_trim
#pragma weak rbk_group_trim

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
  rbk_status append_f64(const double* rows, int64_t n, int64_t* first) {
    return grp ? rbk_group_append_f64(grp, rows, n, first) : rbk_index_append_f64(ix, rows, n, first);
  }
  rbk_status overwrite_batch(const int64_t* slots, int64_t n, const double* rows) {
    return grp ? rbk_group_overwrite_f64_batch(grp, slots, n, rows) : rbk_index_overwrite_f64_batch(ix, slots, n, rows);
  }
  rbk_status tombstone(const int64_t* slots, int64_t n) {
    return grp ? rbk_group_tombstone(grp, slots, n) : rbk_index_tombstone(ix, slots, n);
  }
  rbk_status clear() { return grp ? rbk_group_clear(grp) : rbk_index_clear(ix); }
  bool has_trim() const { return grp ? rbk_group_trim != nullptr : rbk_index_trim != nullptr; }
  rbk_status trim() { return grp ? rbk_group_trim(grp) : rbk_index_trim(ix); }
  int64_t count() const { return grp ? rbk_group_count(grp) : rbk_index_count(ix); }
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

napi_value New(napi_env env, napi_callback_info info) {
  size_t argc = 4;
  napi_value argv[4], self;
  NAPI_OK(napi_get_cb_info(env, info, &argc, argv, &self, nullptr));
  int32_t dim = 0, device = 0, host_rows = 0;
  int64_t hint = 0;
  NAPI_OK(napi_get_value_int32(env, argv[0], &dim));
  if (argc > 2) napi_get_value_int64(env, argv[2], &hint);
  if (argc > 3) napi_get_value_int32(env, argv[3], &host_rows);
  Handle* h = new Handle();
  h->dim = dim;
  bool is_array = false;
  if (argc > 1) napi_is_array(env, argv[1], &is_array);
  // KEEP_F64: the reference stores float64 embeddings; keep them so results are exact for any input.  hostRows
  // (RUNBOOK_KNN_F64_ON_HOST in ts/gpu-embedding-index.ts): keep them in pinned host memory instead of on the GPU.
  const uint32_t flags = RBK_INDEX_KEEP_F64 | (host_rows != 0 ? RBK_INDEX_F64_ON_HOST : 0u);
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
// old_to_new[s] (-1 = it was deleted).  Synchronous.  Single-device handles only.
napi_value Compact(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  if (h->grp) {
    napi_throw_error(env, nullptr, "compaction is not available for a device group");
    return nullptr;
  }
  if (rbk_index_compact == nullptr || rbk_index_size == nullptr) {
    napi_throw_error(env, nullptr, "compact: this librbk_knn.so has no compaction (rbk_index_compact)");
    return nullptr;
  }
  const int64_t n = rbk_index_size(h->ix);
  napi_value ab, out;
  void* p = nullptr;
  NAPI_OK(napi_create_arraybuffer(env, (size_t)n * 8, &p, &ab));
  if (rbk_index_compact(h->ix, static_cast<int64_t*>(p), n) != RBK_OK) return throw_rbk(env);
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

napi_value Count(napi_env env, napi_callback_info info) {
  size_t argc = 0;
  Handle* h = unwrap(env, info, &argc, nullptr);
  napi_value out;
  NAPI_OK(napi_create_int64(env, h->count(), &out));
  return out;
}

// ---- search: runs on a libuv worker so the JS thread never blocks on the GPU ----
enum class SearchKind { kScan, kLarge, kUnbounded };   // search / searchLarge / searchUnbounded

struct SearchJob {
  Handle* ix;
  std::vector<double> queries;
  int32_t B, dim, k;
  SearchKind kind;
  double min_score;
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
  napi_typedarray_type t;
  size_t len;
  void* data;
  NAPI_OK(napi_get_typedarray_info(env, argv[0], &t, &len, &data, nullptr, nullptr));
  auto* j = new SearchJob();
  j->ix = ix;
  j->kind = kind;
  napi_get_value_int32(env, argv[1], &j->B);
  napi_get_value_int32(env, argv[2], &j->k);
  napi_get_value_double(env, argv[3], &j->min_score);   // pass -Infinity for "no threshold"
  j->dim = j->B > 0 ? (int32_t)(len / (size_t)j->B) : 0;   // a wrong length surfaces as RBK_EDIM
  j->queries.assign(static_cast<double*>(data), static_cast<double*>(data) + len);
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
      {"count", nullptr, Count, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"search", nullptr, Search, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"searchLarge", nullptr, SearchLarge, nullptr, nullptr, nullptr, napi_default, nullptr},
      {"searchUnbounded", nullptr, SearchUnbounded, nullptr, nullptr, nullptr, napi_default, nullptr},
  };
  napi_value cls;
  NAPI_OK(napi_define_class(env, "RbkIndex", NAPI_AUTO_LENGTH, New, nullptr, sizeof props / sizeof props[0], props, &cls));
  NAPI_OK(napi_set_named_property(env, exports, "RbkIndex", cls));
  return exports;
}

}  // namespace

NAPI_MODULE(NODE_GYP_MODULE_NAME, Init)
