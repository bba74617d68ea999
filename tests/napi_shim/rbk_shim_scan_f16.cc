// rbk_shim_scan_f16.cc - TEST INFRASTRUCTURE: the oracle-backed CPU stand-in of rbk_shim.cc whose two constructors
// report the flags they were given ("create_ex flags <n>" / "group_create flags <n>" on stderr) and check them as the
// library does, RBK_INDEX_SCAN_F16 included.  Lets tests/test_scan_f16_host.py see which flags the addon's scanF16
// argument asks for where there is no GPU.  Never part of the product.
#include <stdio.h>

#define rbk_index_create_ex shim_base_index_create_ex
#define rbk_group_create shim_base_group_create
#include "rbk_shim.cc"
#undef rbk_index_create_ex
#undef rbk_group_create

namespace {
rbk_status check_flags(uint32_t flags) {
  if (flags & ~static_cast<uint32_t>(RBK_INDEX_KEEP_F64 | RBK_INDEX_F64_ON_HOST | RBK_INDEX_SCAN_F16))
    return fail(RBK_EINVAL, "unknown flag");
  if ((flags & RBK_INDEX_F64_ON_HOST) && !(flags & RBK_INDEX_KEEP_F64))
    return fail(RBK_EINVAL, "RBK_INDEX_F64_ON_HOST requires RBK_INDEX_KEEP_F64");
  if ((flags & RBK_INDEX_SCAN_F16) && !(flags & RBK_INDEX_KEEP_F64))
    return fail(RBK_EINVAL, "RBK_INDEX_SCAN_F16 requires RBK_INDEX_KEEP_F64");
  return RBK_OK;
}
}  // namespace

extern "C" {

rbk_status rbk_index_create_ex(int32_t dim, int32_t device, int64_t hint, uint32_t flags, rbk_index** out) {
  fprintf(stderr, "create_ex flags %u\n", flags);
  const rbk_status st = check_flags(flags);
  return st != RBK_OK ? st : shim_base_index_create_ex(dim, device, hint, flags, out);
}

rbk_status rbk_group_create(int32_t dim, const int32_t* device_ids, int32_t n_devices, int64_t hint, uint32_t flags,
                            rbk_group** out) {
  fprintf(stderr, "group_create flags %u\n", flags);
  const rbk_status st = check_flags(flags);
  return st != RBK_OK ? st : shim_base_group_create(dim, device_ids, n_devices, hint, flags, out);
}

}  // extern "C"
