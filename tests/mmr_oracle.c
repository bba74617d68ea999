/*
 * mmr_oracle.c — TEST INFRASTRUCTURE: the greedy selection of maximal marginal relevance, restated from the contract
 * of rbk_index_search_mmr_f64 (include/rbk_knn.h), not from the kernel.  Built by tests/mmr_oracle.py with the
 * oracle's flags (-O2 -ffp-contract=off, no fast-math) and linked against the oracle's rbk_oracle_cosine, the
 * reference's cosineSimilarity; tests/napi_shim/rbk_shim_mmr.cc compiles it into the addon's CPU stand-in.  Valid C and
 * C++.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

double rbk_oracle_cosine(const double *a, const double *b, int64_t d);

/* rows [m][d]: the stored values of candidates c_0 .. c_{m-1}; r [m]: their relevance.  Writes the candidate indices of
 * the min(k, m) picks, in selection order, to picks and returns how many there are (-1: out of memory). */
int64_t rbk_oracle_mmr_select(const double *rows, int64_t m, int64_t d, const double *r, int64_t k, double lam,
                              int64_t *picks) {
  const int64_t n = k < m ? k : m;
  if (n <= 0) return 0;
  double *red = (double *)malloc(sizeof(double) * (size_t)m);
  unsigned char *picked = (unsigned char *)calloc((size_t)m, 1);
  if (!red || !picked) {
    free(red);
    free(picked);
    return -1;
  }
  for (int64_t i = 0; i < m; i++) red[i] = NAN;
  picks[0] = 0; /* the first pick is c_0 */
  picked[0] = 1;
  for (int64_t t = 1; t < n; t++) {
    const double *last = rows + picks[t - 1] * d;
    int64_t best = -1;
    double best_v = 0.0;
    for (int64_t i = 0; i < m; i++) {
      if (picked[i]) continue;
      const double s = rbk_oracle_cosine(rows + i * d, last, d);
      if (isnan(red[i]) || s > red[i]) red[i] = s; /* the largest non-NaN s so far, NaN while every s was NaN */
      const double one_minus = 1.0 - lam;
      const double a = lam * r[i];
      const double c = one_minus * red[i];
      const double v = a - c;
      /* a NaN ranks below every number, then the larger value, then the smaller index (i ascends: strictly better) */
      if (best < 0 || (!isnan(v) && (isnan(best_v) || v > best_v))) {
        best = i;
        best_v = v;
      }
    }
    picks[t] = best;
    picked[best] = 1;
  }
  free(red);
  free(picked);
  return n;
}
