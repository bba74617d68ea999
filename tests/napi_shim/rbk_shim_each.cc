// rbk_shim_each.cc - TEST INFRASTRUCTURE: the oracle-backed CPU stand-in of rbk_shim_unbounded.cc plus the per-query
// entry points (rbk_index_search_each_f64 / rbk_group_search_each_f64): each query answered by the same oracle call at
// its own k_fetch and min_score, rows of max k_fetch entries.  Lets tests/test_search_each_host.py run the addon's
// searchEach where there is no GPU.  Never part of the product.
#include "rbk_shim_unbounded.cc"

#include <string>

extern "C" {

rbk_status rbk_index_search_each_f64(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim,
                                     const int32_t* k_fetch, const double* min_score, int64_t* out_slots,
                                     double* out_scores, int32_t* out_counts, float*) {
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  if (B > 0 && (!queries || !k_fetch || !min_score)) return fail(RBK_EINVAL, "null k_fetch or min_score array");
  int32_t K = 0;
  for (int32_t b = 0; b < B; ++b) {
    if (k_fetch[b] < 1) return fail(RBK_EINVAL, ("k_fetch[" + std::to_string(b) + "] must be >= 1").c_str());
    K = k_fetch[b] > K ? k_fetch[b] : K;
  }
  if (query_dim != ix->dim) return fail(RBK_EDIM, "Vectors must have the same length");
  for (int32_t b = 0; b < B; ++b) {
    if (min_score[b] != min_score[b]) return fail(RBK_EINVAL, ("min_score[" + std::to_string(b) + "] is NaN").c_str());
  }
  for (int32_t b = 0; b < B; ++b) {
    int64_t* s = out_slots + static_cast<size_t>(b) * K;
    double* v = out_scores + static_cast<size_t>(b) * K;
    for (int32_t i = 0; i < K; ++i) {
      s[i] = -1;
      const uint64_t nan_bits = 0x7FF8000000000000ull;
      memcpy(&v[i], &nan_bits, 8);
    }
    out_counts[b] = static_cast<int32_t>(rbk_oracle_search_f64(ix->rows.data(), static_cast<int64_t>(ix->live.size()),
                                                               ix->dim, queries + static_cast<size_t>(b) * ix->dim,
                                                               ix->dim, ix->live.data(), 1, min_score[b], k_fetch[b],
                                                               s, v));
  }
  return RBK_OK;
}

rbk_status rbk_group_search_each_f64(rbk_group* g, const double* queries, int32_t B, int32_t query_dim,
                                     const int32_t* k_fetch, const double* min_score, int64_t* out_slots,
                                     double* out_scores, int32_t* out_counts, float* ms) {
  return rbk_index_search_each_f64(&g->ix, queries, B, query_dim, k_fetch, min_score, out_slots, out_scores,
                                   out_counts, ms);
}

}  // extern "C"
