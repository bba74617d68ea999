// rbk_shim_slots.cc - TEST INFRASTRUCTURE: the oracle-backed CPU stand-in of rbk_shim_each.cc plus stored rows as
// queries (rbk_index_search_slots_f64 / rbk_group_search_slots_f64): the search_each of the stand-in on the rows of the
// named slots.  Lets tests/test_search_slots_host.py run the addon's searchSlots where there is no GPU.  Never part of
// the product.
#include "rbk_shim_each.cc"

#include <string>
#include <vector>

extern "C" {

rbk_status rbk_index_search_slots_f64(rbk_index* ix, const int64_t* query_slots, int32_t B, const int32_t* k_fetch,
                                      const double* min_score, int64_t* out_slots, double* out_scores,
                                      int32_t* out_counts, float* ms) {
  if (B > 0 && !query_slots) return fail(RBK_EINVAL, "bad queries argument");
  std::vector<double> q(static_cast<size_t>(B > 0 ? B : 0) * ix->dim);
  for (int32_t b = 0; b < B; ++b) {
    const int64_t s = query_slots[b];
    if (s < 0 || s >= static_cast<int64_t>(ix->live.size()))
      return fail(RBK_EINVAL, ("query_slots[" + std::to_string(b) + "] is not a slot of this index").c_str());
    if (!ix->live[s]) return fail(RBK_EINVAL, "query slot is tombstoned (1 of the batch)");
    memcpy(q.data() + static_cast<size_t>(b) * ix->dim, ix->rows.data() + static_cast<size_t>(s) * ix->dim,
           sizeof(double) * ix->dim);
  }
  return rbk_index_search_each_f64(ix, q.data(), B, ix->dim, k_fetch, min_score, out_slots, out_scores, out_counts,
                                   ms);
}

rbk_status rbk_group_search_slots_f64(rbk_group* g, const int64_t* query_slots, int32_t B, const int32_t* k_fetch,
                                      const double* min_score, int64_t* out_slots, double* out_scores,
                                      int32_t* out_counts, float* ms) {
  return rbk_index_search_slots_f64(&g->ix, query_slots, B, k_fetch, min_score, out_slots, out_scores, out_counts, ms);
}

}  // extern "C"
