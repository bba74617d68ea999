// rbk_shim_mmr.cc - TEST INFRASTRUCTURE: the oracle-backed CPU stand-in of rbk_shim_each.cc plus diverse hits by
// maximal marginal relevance (rbk_index_search_mmr_f64 / rbk_group_search_mmr_f64): each query's candidates from the
// oracle's search at its fetch_k, the greedy selection of tests/mmr_oracle.c on their rows.  Lets
// tests/test_mmr_host.py run the addon's searchMmr where there is no GPU.  Never part of the product.
#include "rbk_shim_each.cc"

#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include <string>
#include <vector>

extern "C" {
#include "../mmr_oracle.c"

rbk_status rbk_index_search_mmr_f64(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim,
                                    const int32_t* k, const int32_t* fetch_k, const double* lambda_mult,
                                    const double* min_score, int64_t* out_slots, double* out_scores,
                                    int32_t* out_counts, float*) {
  if (B > 0 && (!queries || !k || !fetch_k || !lambda_mult || !min_score))
    return fail(RBK_EINVAL, "null k, fetch_k, lambda_mult or min_score array");
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  int32_t K = 0;
  for (int32_t b = 0; b < B; ++b) {
    const std::string at = "[" + std::to_string(b) + "]";
    if (k[b] < 1) return fail(RBK_EINVAL, ("k" + at + " must be >= 1").c_str());
    if (fetch_k[b] < k[b]) return fail(RBK_EINVAL, ("fetch_k" + at + " must be >= k" + at).c_str());
    if (fetch_k[b] > RBK_MAX_K_FETCH_LARGE) return fail(RBK_EINVAL, ("fetch_k" + at + " must be <= 4096").c_str());
    if (static_cast<int64_t>(fetch_k[b]) * ix->dim > RBK_MMR_MAX_FETCH_ELEMS)
      return fail(RBK_EINVAL, ("fetch_k" + at + " * dim must be <= RBK_MMR_MAX_FETCH_ELEMS").c_str());
    K = k[b] > K ? k[b] : K;
  }
  if (query_dim != ix->dim) return fail(RBK_EDIM, "Vectors must have the same length");
  for (int32_t b = 0; b < B; ++b) {
    if (min_score[b] != min_score[b]) return fail(RBK_EINVAL, ("min_score[" + std::to_string(b) + "] is NaN").c_str());
    if (!(lambda_mult[b] >= 0.0 && lambda_mult[b] <= 1.0))
      return fail(RBK_EINVAL, ("lambda_mult[" + std::to_string(b) + "] must be in [0, 1]").c_str());
  }
  const int64_t n = static_cast<int64_t>(ix->live.size());
  for (int32_t b = 0; b < B; ++b) {
    std::vector<int64_t> cs(fetch_k[b]), picks(k[b]);
    std::vector<double> cv(fetch_k[b]);
    const int64_t m = rbk_oracle_search_f64(ix->rows.data(), n, ix->dim, queries + static_cast<size_t>(b) * ix->dim,
                                            ix->dim, ix->live.data(), 1, min_score[b], fetch_k[b], cs.data(), cv.data());
    std::vector<double> rows(static_cast<size_t>(m) * ix->dim);
    for (int64_t i = 0; i < m; ++i)
      memcpy(&rows[i * ix->dim], &ix->rows[cs[i] * ix->dim], sizeof(double) * ix->dim);
    const int64_t c = rbk_oracle_mmr_select(rows.data(), m, ix->dim, cv.data(), k[b], lambda_mult[b], picks.data());
    if (c < 0) return fail(RBK_ENOMEM, "out of memory");
    int64_t* s = out_slots + static_cast<size_t>(b) * K;
    double* v = out_scores + static_cast<size_t>(b) * K;
    const uint64_t nan_bits = 0x7FF8000000000000ull;
    for (int32_t i = 0; i < K; ++i) {
      s[i] = i < c ? cs[picks[i]] : -1;
      if (i < c) v[i] = cv[picks[i]];
      else memcpy(&v[i], &nan_bits, 8);
    }
    out_counts[b] = static_cast<int32_t>(c);
  }
  return RBK_OK;
}

rbk_status rbk_group_search_mmr_f64(rbk_group* g, const double* queries, int32_t B, int32_t query_dim,
                                    const int32_t* k, const int32_t* fetch_k, const double* lambda_mult,
                                    const double* min_score, int64_t* out_slots, double* out_scores,
                                    int32_t* out_counts, float* ms) {
  return rbk_index_search_mmr_f64(&g->ix, queries, B, query_dim, k, fetch_k, lambda_mult, min_score, out_slots,
                                  out_scores, out_counts, ms);
}

}  // extern "C"
