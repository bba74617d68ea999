// rbk_shim_group_compact.cc - TEST INFRASTRUCTURE: the oracle-backed CPU stand-in of rbk_shim_compact.cc plus
// rbk_group_size and rbk_group_compact.  The stand-in's group is one host index in global slot order, so compacting
// it is rbk_index_compact's contract in global slots.  Lets tests/test_group_compact_host.py run the addon's compact()
// on a device-group handle where there is no GPU.  Never part of the product.
#include "rbk_shim_compact.cc"

extern "C" {

int64_t rbk_group_size(const rbk_group* g) { return g ? rbk_index_size(&g->ix) : 0; }

rbk_status rbk_group_compact(rbk_group* g, int64_t* old_to_new, int64_t old_to_new_len) {
  if (!g) return fail(RBK_EINVAL, "null group");
  return rbk_index_compact(&g->ix, old_to_new, old_to_new_len);
}

}  // extern "C"
