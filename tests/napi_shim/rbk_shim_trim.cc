// rbk_shim_trim.cc - TEST INFRASTRUCTURE: the oracle-backed CPU stand-in of rbk_shim.cc plus rbk_index_trim and
// rbk_group_trim.  The stand-in has no device memory to give back, so a trim changes nothing; each call prints one
// line to stderr, so that tests/test_trim_host.py can see which entry point the addon's trim() reached.  Never part of
// the product.
#include <stdio.h>

#include "rbk_shim.cc"

extern "C" {

rbk_status rbk_index_trim(rbk_index* ix) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  fprintf(stderr, "rbk_shim: rbk_index_trim\n");
  return RBK_OK;
}

rbk_status rbk_group_trim(rbk_group* g) {
  if (!g) return fail(RBK_EINVAL, "null group");
  fprintf(stderr, "rbk_shim: rbk_group_trim\n");
  return RBK_OK;
}

}  // extern "C"
