// rbk_shim_pairs.cc - TEST INFRASTRUCTURE: the oracle-backed CPU stand-in of rbk_shim_slots.cc plus every pair above a
// threshold (rbk_index_similar_pairs_f64 / rbk_group_similar_pairs_f64): for each live row a from first_slot on, the
// stand-in's search_slots({a}, count(), min_score) above a, whole rows while they fit in max_pairs.  Lets
// tests/test_similar_pairs_host.py run the addon's similarPairs where there is no GPU.  Never part of the product.
#include "rbk_shim_slots.cc"

#include <string>
#include <vector>

extern "C" {

rbk_status rbk_index_similar_pairs_f64(rbk_index* ix, double min_score, int64_t first_slot, int64_t max_pairs,
                                       int64_t* out_a, int64_t* out_b, double* out_scores, int64_t* n_out,
                                       int64_t* next_slot, float*) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  if (!out_a || !out_b || !out_scores || !n_out || !next_slot) return fail(RBK_EINVAL, "null output");
  if (min_score != min_score) return fail(RBK_EINVAL, "min_score is NaN");
  const int64_t size = static_cast<int64_t>(ix->live.size());
  if (first_slot < 0 || first_slot > size) return fail(RBK_EINVAL, "first_slot must be in [0, size()]");
  if (max_pairs < (size > 1 ? size : 1)) return fail(RBK_EINVAL, "max_pairs must be >= max(size(), 1)");
  int32_t count = 0;
  for (uint8_t l : ix->live) count += l;
  int64_t n = 0, a = first_slot;
  std::vector<int64_t> s(count > 0 ? count : 1);
  std::vector<double> v(s.size());
  for (; a < size; ++a) {
    if (!ix->live[a]) continue;
    int32_t c = 0;
    rbk_status st = rbk_index_search_slots_f64(ix, &a, 1, &count, &min_score, s.data(), v.data(), &c, nullptr);
    if (st != RBK_OK) return st;
    int64_t k = 0;
    for (int32_t i = 0; i < c; ++i) k += s[i] > a;
    if (n + k > max_pairs) break;
    for (int32_t i = 0; i < c; ++i)
      if (s[i] > a) {
        out_a[n] = a;
        out_b[n] = s[i];
        out_scores[n++] = v[i];
      }
  }
  *n_out = n;
  *next_slot = a;
  return RBK_OK;
}

rbk_status rbk_group_similar_pairs_f64(rbk_group* g, double min_score, int64_t first_slot, int64_t max_pairs,
                                       int64_t* out_a, int64_t* out_b, double* out_scores, int64_t* n_out,
                                       int64_t* next_slot, float* ms) {
  return rbk_index_similar_pairs_f64(g ? &g->ix : nullptr, min_score, first_slot, max_pairs, out_a, out_b, out_scores,
                                     n_out, next_slot, ms);
}

}  // extern "C"
