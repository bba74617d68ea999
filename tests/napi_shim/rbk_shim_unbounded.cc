// rbk_shim_unbounded.cc - TEST INFRASTRUCTURE: the oracle-backed CPU stand-in of rbk_shim_large.cc plus the unbounded
// entry points (rbk_index_search_unbounded_f64 / rbk_group_search_unbounded_f64), answered by the same oracle call,
// which takes any k_fetch.  Lets tests/test_unbounded_host.py run the addon's searchUnbounded where there is no GPU.
// Never part of the product.
#include "rbk_shim_large.cc"

extern "C" {

rbk_status rbk_index_search_unbounded_f64(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim,
                                          int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                          int32_t* out_counts, float*) {
  if (k_fetch < 1) return fail(RBK_EINVAL, "k_fetch must be in [1, 2147483647]");
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

rbk_status rbk_group_search_unbounded_f64(rbk_group* g, const double* queries, int32_t B, int32_t query_dim,
                                          int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                          int32_t* out_counts, float* ms) {
  return rbk_index_search_unbounded_f64(&g->ix, queries, B, query_dim, k_fetch, min_score, out_slots, out_scores,
                                        out_counts, ms);
}

}  // extern "C"
