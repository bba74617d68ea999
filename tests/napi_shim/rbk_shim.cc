// rbk_shim.cc - TEST INFRASTRUCTURE: a CPU stand-in for the handful of librbk_knn.so entry points that
// napi/rbk_napi.cc binds, answered by the oracle (oracle/librbk_oracle.so).  It exists so that the addon + mock
// N-API harness (napi/mock/) can run its whole scenario on a box without a GPU and be compared with the oracle;
// the `-m gpu` test links the same harness against the real library instead.  Never part of the product.
#include <string.h>

#include <string>
#include <vector>

#include "../../include/rbk_knn.h"

extern "C" int64_t rbk_oracle_search_f64(const double* corpus, int64_t n, int64_t d, const double* q, int64_t qd,
                                         const uint8_t* live, int use_threshold, double min_score, int64_t k_fetch,
                                         int64_t* out_slots, double* out_scores);

struct rbk_index {
  int32_t dim = 0;
  std::vector<double> rows;
  std::vector<uint8_t> live;
};
struct rbk_group {
  rbk_index ix;
};

namespace {
thread_local std::string g_err;
rbk_status fail(rbk_status st, const char* msg) {
  g_err = msg;
  return st;
}
}  // namespace

extern "C" {

const char* rbk_last_error(void) { return g_err.c_str(); }
int rbk_abi_version(void) { return RBK_ABI_VERSION; }

rbk_status rbk_index_create_ex(int32_t dim, int32_t device, int64_t, uint32_t, rbk_index** out) {
  if (dim < 1 || dim > RBK_MAX_DIM) return fail(RBK_EINVAL, "dim out of range");
  if (device != 0) return fail(RBK_EINVAL, "device ordinal out of range");
  *out = new rbk_index();
  (*out)->dim = dim;
  return RBK_OK;
}
void rbk_index_destroy(rbk_index* ix) { delete ix; }

rbk_status rbk_index_append_f64(rbk_index* ix, const double* rows, int64_t n, int64_t* first) {
  if (first) *first = static_cast<int64_t>(ix->live.size());
  ix->rows.insert(ix->rows.end(), rows, rows + n * ix->dim);
  ix->live.insert(ix->live.end(), static_cast<size_t>(n), 1);
  return RBK_OK;
}
rbk_status rbk_index_overwrite_f64_batch(rbk_index* ix, const int64_t* slots, int64_t n, const double* rows) {
  int dead = 0;
  for (int64_t i = 0; i < n; ++i)
    if (slots[i] < 0 || slots[i] >= static_cast<int64_t>(ix->live.size())) return fail(RBK_EINVAL, "slot out of range");
  for (int64_t i = 0; i < n; ++i) {
    if (!ix->live[slots[i]]) {
      dead++;
      continue;
    }
    memcpy(&ix->rows[slots[i] * ix->dim], rows + i * ix->dim, sizeof(double) * ix->dim);
  }
  return dead ? fail(RBK_EINVAL, "slot is tombstoned") : RBK_OK;
}
rbk_status rbk_index_tombstone(rbk_index* ix, const int64_t* slots, int64_t n) {
  for (int64_t i = 0; i < n; ++i)
    if (slots[i] < 0 || slots[i] >= static_cast<int64_t>(ix->live.size())) return fail(RBK_EINVAL, "slot out of range");
  for (int64_t i = 0; i < n; ++i) ix->live[slots[i]] = 0;
  return RBK_OK;
}
rbk_status rbk_index_clear(rbk_index* ix) {
  ix->rows.clear();
  ix->live.clear();
  return RBK_OK;
}
int64_t rbk_index_count(const rbk_index* ix) {
  int64_t c = 0;
  for (uint8_t l : ix->live) c += l;
  return c;
}
rbk_status rbk_index_search_f64(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                                double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts, float*) {
  if (k_fetch < 1 || k_fetch > RBK_MAX_K_FETCH) return fail(RBK_EINVAL, "k_fetch must be in [1, 112]");
  if (query_dim != ix->dim) return fail(RBK_EDIM, "Vectors must have the same length");
  for (int32_t b = 0; b < B; ++b) {
    for (int32_t i = 0; i < k_fetch; ++i) {
      out_slots[static_cast<size_t>(b) * k_fetch + i] = -1;
      memset(&out_scores[static_cast<size_t>(b) * k_fetch + i], 0xFF, 8);
    }
    out_counts[b] = static_cast<int32_t>(rbk_oracle_search_f64(
        ix->rows.data(), static_cast<int64_t>(ix->live.size()), ix->dim, queries + static_cast<size_t>(b) * ix->dim,
        ix->dim, ix->live.data(), 1, min_score, k_fetch, out_slots + static_cast<size_t>(b) * k_fetch,
        out_scores + static_cast<size_t>(b) * k_fetch));
  }
  return RBK_OK;
}

// the group family: same behaviour behind the other handle type (global slots = insertion order)
rbk_status rbk_group_create(int32_t dim, const int32_t* device_ids, int32_t n_devices, int64_t, uint32_t, rbk_group** out) {
  if (!device_ids || n_devices < 1) return fail(RBK_EINVAL, "bad device list");
  if (dim < 1 || dim > RBK_MAX_DIM) return fail(RBK_EINVAL, "dim out of range");
  *out = new rbk_group();
  (*out)->ix.dim = dim;
  return RBK_OK;
}
void rbk_group_destroy(rbk_group* g) { delete g; }
rbk_status rbk_group_append_f64(rbk_group* g, const double* rows, int64_t n, int64_t* first) {
  return rbk_index_append_f64(&g->ix, rows, n, first);
}
rbk_status rbk_group_overwrite_f64_batch(rbk_group* g, const int64_t* slots, int64_t n, const double* rows) {
  return rbk_index_overwrite_f64_batch(&g->ix, slots, n, rows);
}
rbk_status rbk_group_tombstone(rbk_group* g, const int64_t* slots, int64_t n) {
  return rbk_index_tombstone(&g->ix, slots, n);
}
rbk_status rbk_group_clear(rbk_group* g) { return rbk_index_clear(&g->ix); }
int64_t rbk_group_count(const rbk_group* g) { return rbk_index_count(&g->ix); }
rbk_status rbk_group_search_f64(rbk_group* g, const double* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                                double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts, float* ms) {
  return rbk_index_search_f64(&g->ix, queries, B, query_dim, k_fetch, min_score, out_slots, out_scores, out_counts, ms);
}

}  // extern "C"
