// rbk_shim_compact.cc - TEST INFRASTRUCTURE: the oracle-backed CPU stand-in of rbk_shim.cc plus rbk_index_size and
// rbk_index_compact, done on the stand-in's host rows with the library's contract (live rows keep their order,
// old_to_new = new slot or -1).  Lets tests/test_compact_host.py run the addon's compact() where there is no GPU.
// Never part of the product.
#include "rbk_shim.cc"

extern "C" {

int64_t rbk_index_size(const rbk_index* ix) { return ix ? static_cast<int64_t>(ix->live.size()) : 0; }

rbk_status rbk_index_compact(rbk_index* ix, int64_t* old_to_new, int64_t old_to_new_len) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  const int64_t n = static_cast<int64_t>(ix->live.size());
  if (old_to_new && old_to_new_len < n) return fail(RBK_EINVAL, "old_to_new_len is shorter than size()");
  int64_t next = 0;
  for (int64_t s = 0; s < n; ++s) {
    const int64_t to = ix->live[s] ? next++ : -1;
    if (old_to_new) old_to_new[s] = to;
    if (to >= 0 && to != s) memcpy(&ix->rows[to * ix->dim], &ix->rows[s * ix->dim], sizeof(double) * ix->dim);
  }
  ix->rows.resize(static_cast<size_t>(next) * ix->dim);
  ix->live.assign(static_cast<size_t>(next), 1);
  return RBK_OK;
}

}  // extern "C"
