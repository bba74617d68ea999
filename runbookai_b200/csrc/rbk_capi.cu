// rbk_capi.cu — the C ABI of include/rbk_knn.h: index lifetime, mutation, batched search.
// Host-side orchestration only; the device work is in rbk_ingest.cu / rbk_scan.cu /
// rbk_finalize.cu.  No torch, no CPU compute path: every entry point that needs a GPU
// fails with RBK_ECUDA when there is none.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "rbk_index_impl.h"

using namespace rbk;

namespace rbk {
namespace impl {
thread_local std::string g_err_storage;
rbk_status fail(rbk_status st, const std::string& msg) {
  g_err_storage = msg;
  return st;
}
rbk_status cuda_fail(cudaError_t e, const char* what) {
  // a sticky error (trap in a kernel) poisons the context; report it verbatim
  return fail(e == cudaErrorMemoryAllocation ? RBK_ENOMEM : RBK_ECUDA,
              std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")");
}
const char* last_error() { return g_err_storage.c_str(); }
}  // namespace impl
}  // namespace rbk
using namespace rbk::impl;

// fill_empty_results' slots and scores (outside the anonymous namespaces: nvcc's host stub for a kernel inside one
// cannot tell this file's several apart)
static __global__ void empty_results_kernel(long long* slots, double* scores, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    slots[i] = -1;
    scores[i] = __longlong_as_double(0x7FF8000000000000ll);
  }
}

namespace {


typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// 2D bf16 (f16: fp16) row-major [rows][dpad] tensor, box = box_cols columns (one swizzle row: 64 -> 128 B, 32 -> 64 B)
// x box_rows.
rbk_status encode_rows_tmap(CUtensorMap* out, const void* base, int64_t rows, int dpad, int box_rows, bool f16,
                            int box_cols = kBlockK) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(RBK_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(dpad), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(dpad) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  box_cols == 32 ? CU_TENSOR_MAP_SWIZZLE_64B
                                 : (box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE),
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed: CUresult %d (rows=%lld dpad=%d)", (int)r,
             (long long)rows, dpad);
    return fail(RBK_ECUDA, buf);
  }
  return RBK_OK;
}

int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// Page-locked (or managed) host memory: cudaMemcpyAsync from it returns before the bytes have been read, unlike a copy
// from pageable memory, which the driver stages before returning.
bool host_source_is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

// Fold finished (start, stop) pairs into the running totals.  wait = true: block on the pending ones.
void resolve_scan_events(rbk_index* ix, bool wait) {
  while (ix->tev_tail < ix->tev_head) {
    cudaEvent_t* pr = ix->tev[ix->tev_tail % rbk_index::kTimingRing];
    if (wait) cudaEventSynchronize(pr[1]);
    else if (cudaEventQuery(pr[1]) != cudaSuccess) { cudaGetLastError(); break; }
    float t = 0.f;
    if (cudaEventElapsedTime(&t, pr[0], pr[1]) == cudaSuccess) {
      ix->stats.scan_ms_total += t;
      ix->stats.scans_timed++;
      ix->stats.last_scan_ms = t;
    }
    ix->tev_tail++;
  }
}
// Next (start, stop) pair of the ring; created on first use.
cudaEvent_t* next_scan_events(rbk_index* ix) {
  if (ix->tev_head - ix->tev_tail >= rbk_index::kTimingRing) {   // ring full: the oldest finished long ago
    cudaEvent_t* old = ix->tev[ix->tev_tail % rbk_index::kTimingRing];
    cudaEventSynchronize(old[1]);
    resolve_scan_events(ix, false);
  }
  cudaEvent_t* pr = ix->tev[ix->tev_head % rbk_index::kTimingRing];
  if (!pr[0]) {
    cudaEventCreate(&pr[0]);
    cudaEventCreate(&pr[1]);
  }
  ix->tev_head++;
  return pr;
}

int64_t inv_norm_len(int64_t cap) { return round_up(cap, kBlockN) + kBlockN; }

// ---- device corpus storage on reserved virtual address ranges (DESIGN.md §3) ----
// The driver's virtual memory calls, looked up like cuTensorMapEncodeTiled so that the link line stays the runtime's.
struct VmmApi {
  bool ok = false;
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
};

const VmmApi& vmm_api() {
  static VmmApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    bool ok = true;
    auto get = [&ok](const char* name, auto* fn) {
      void* p = nullptr;
      cudaDriverEntryPointQueryResult qres;
      if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &qres) == cudaSuccess &&
          qres == cudaDriverEntryPointSuccess && p)
        *fn = reinterpret_cast<std::remove_pointer_t<decltype(fn)>>(p);
      else
        ok = false;
    };
    get("cuDeviceGetAttribute", &api.DeviceGetAttribute);
    get("cuMemGetAllocationGranularity", &api.MemGetAllocationGranularity);
    get("cuMemAddressReserve", &api.MemAddressReserve);
    get("cuMemAddressFree", &api.MemAddressFree);
    get("cuMemCreate", &api.MemCreate);
    get("cuMemRelease", &api.MemRelease);
    get("cuMemMap", &api.MemMap);
    get("cuMemUnmap", &api.MemUnmap);
    get("cuMemSetAccess", &api.MemSetAccess);
    api.ok = ok;
  });
  return api;
}

rbk_status cu_fail(CUresult r, const char* what) {
  return fail(r == CUDA_ERROR_OUT_OF_MEMORY ? RBK_ENOMEM : RBK_ECUDA,
              std::string(what) + " failed: CUresult " + std::to_string(static_cast<int>(r)));
}

CUmemAllocationProp vm_prop(int device) {
  CUmemAllocationProp prop;
  memset(&prop, 0, sizeof prop);
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  return prop;
}

// Largest physical chunk of one mapping.  A growth maps [old, new) of a buffer in chunks of at most this size (one
// chunk when the growth is smaller), so growing to a full 80 GB card takes a few hundred map calls, a small index pays
// one granule (2 MiB on H100) per small buffer, and a trim leaves less than one chunk per buffer mapped beyond the
// capacity (DESIGN.md §3).
constexpr size_t kVmChunk = 256ull << 20;

// Unmaps and releases the chunks of r that lie wholly at or beyond `keep` bytes from its base.
void vm_unmap_from(VmRange* r, size_t keep) {
  const VmmApi& api = vmm_api();
  while (!r->chunks.empty() && r->mapped - r->chunks.back().bytes >= keep) {
    const VmRange::Chunk c = r->chunks.back();
    r->mapped -= c.bytes;
    api.MemUnmap(r->base + r->mapped, c.bytes);
    api.MemRelease(c.handle);
    r->chunks.pop_back();
  }
}

// Backs [base, base + bytes) of r, mapping new chunks after the ones it has.  On failure the chunks this call mapped
// stay mapped; the caller unmaps them (vm_unmap_from its old `mapped`).
rbk_status vm_map_to(const rbk_index* ix, VmRange* r, size_t bytes) {
  const VmmApi& api = vmm_api();
  const size_t want = static_cast<size_t>(round_up(static_cast<int64_t>(bytes), static_cast<int64_t>(ix->vm_gran)));
  if (want > r->reserved) return fail(RBK_ENOMEM, "index storage beyond its reserved address range");
  const size_t max_chunk = std::max(ix->vm_gran, kVmChunk / ix->vm_gran * ix->vm_gran);
  const CUmemAllocationProp prop = vm_prop(ix->device);
  CUmemAccessDesc access;
  memset(&access, 0, sizeof access);
  access.location = prop.location;
  access.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  while (r->mapped < want) {
    const size_t sz = std::min(want - r->mapped, max_chunk);
    CUmemGenericAllocationHandle h;
    CUresult res = api.MemCreate(&h, sz, &prop, 0);
    if (res != CUDA_SUCCESS) return cu_fail(res, "cuMemCreate(index storage)");
    const CUdeviceptr at = r->base + r->mapped;
    if ((res = api.MemMap(at, sz, 0, h, 0)) != CUDA_SUCCESS) {
      api.MemRelease(h);
      return cu_fail(res, "cuMemMap(index storage)");
    }
    r->chunks.push_back({h, sz});
    r->mapped += sz;
    if ((res = api.MemSetAccess(at, sz, &access, 1)) != CUDA_SUCCESS) return cu_fail(res, "cuMemSetAccess(index storage)");
  }
  return RBK_OK;
}

// Bytes of each device corpus buffer at capacity `cap` (ix->vm order); 0 for the exact rows unless they live on the
// device (f64_dev: they would, -1: the index's own tier), x_elem bytes per element (-1: the index's own width).
void storage_at(const rbk_index* ix, int64_t cap, size_t out[rbk_index::kVmBuffers], int f64_dev = -1, int x_elem = -1) {
  if (f64_dev < 0) f64_dev = ix->keep_rows() && !ix->rows_on_host;
  if (x_elem < 0) x_elem = ix->x_elem;
  out[0] = static_cast<size_t>(cap) * ix->dpad * 2;
  out[1] = static_cast<size_t>(inv_norm_len(cap)) * 4;
  out[2] = static_cast<size_t>(cap) * 8;
  out[3] = static_cast<size_t>((cap + 31) / 32) * 4;
  out[4] = f64_dev ? static_cast<size_t>(cap) * ix->dim * x_elem : 0;
}

// The most rows the device's memory could back with the exact rows (x_elem bytes per element, -1: the index's own) on
// the device (f64_dev) or not: the row ceiling of a tier, min(2^31 - 512, total memory / device bytes per row) in whole
// tiles.
int64_t tier_vm_rows(const rbk_index* ix, bool f64_dev, int x_elem = -1) {
  // device bytes per row, the tombstone bit rounded up to a byte
  size_t per_row[rbk_index::kVmBuffers];
  storage_at(ix, 1, per_row, f64_dev, x_elem);
  const int64_t row_bytes = static_cast<int64_t>(per_row[0] + 4 + per_row[2] + 1 + per_row[4]);
  return std::min<int64_t>((1ll << 31) - 2 * kBlockN, static_cast<int64_t>(ix->total_mem) / row_bytes / kBlockN * kBlockN);
}

// Backs every device buffer for `ncap` rows: all of them, or (on failure) none of the chunks this call mapped.
rbk_status vm_map_capacity(rbk_index* ix, int64_t ncap) {
  if (ncap > ix->vm_rows)
    return fail(RBK_ENOMEM, "a capacity of " + std::to_string(ncap) + " rows exceeds the " +
                                std::to_string(ix->vm_rows) + " this device can hold");
  size_t want[rbk_index::kVmBuffers], old[rbk_index::kVmBuffers];
  storage_at(ix, ncap, want);
  for (int i = 0; i < rbk_index::kVmBuffers; ++i) old[i] = ix->vm[i].mapped;
  for (int i = 0; i < rbk_index::kVmBuffers; ++i) {
    rbk_status st = vm_map_to(ix, &ix->vm[i], want[i]);
    if (st != RBK_OK) {
      for (int j = 0; j <= i; ++j) vm_unmap_from(&ix->vm[j], old[j]);
      return st;
    }
  }
  return RBK_OK;
}

// Reserves the device buffers' address ranges for the largest capacity the device could back.
rbk_status vm_reserve(rbk_index* ix, size_t total_global_mem) {
  const VmmApi& api = vmm_api();
  if (!api.ok) return fail(RBK_ECUDA, "the driver does not provide the CUDA virtual memory management calls");
  int supported = 0;
  CUresult res = api.DeviceGetAttribute(&supported, CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED, ix->device);
  if (res != CUDA_SUCCESS) return cu_fail(res, "cuDeviceGetAttribute(VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED)");
  if (!supported)
    return fail(RBK_ECUDA, "device " + std::to_string(ix->device) +
                               " does not support CUDA virtual memory management, which the index storage needs");
  const CUmemAllocationProp prop = vm_prop(ix->device);
  if ((res = api.MemGetAllocationGranularity(&ix->vm_gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM)) != CUDA_SUCCESS)
    return cu_fail(res, "cuMemGetAllocationGranularity");
  ix->total_mem = total_global_mem;
  ix->vm_rows = tier_vm_rows(ix, ix->keep_rows() && !ix->rows_on_host);
  size_t bytes[rbk_index::kVmBuffers];
  storage_at(ix, ix->vm_rows, bytes);
  for (int i = 0; i < rbk_index::kVmBuffers; ++i) {
    if (bytes[i] == 0) continue;
    VmRange& r = ix->vm[i];
    const size_t len = static_cast<size_t>(round_up(static_cast<int64_t>(bytes[i]), static_cast<int64_t>(ix->vm_gran)));
    if ((res = api.MemAddressReserve(&r.base, len, 0, 0, 0)) != CUDA_SUCCESS) return cu_fail(res, "cuMemAddressReserve");
    r.reserved = len;
  }
  ix->rows = reinterpret_cast<uint16_t*>(ix->vm[0].base);
  ix->inv_norm = reinterpret_cast<float*>(ix->vm[1].base);
  ix->norm2 = reinterpret_cast<double*>(ix->vm[2].base);
  ix->dead_bits = reinterpret_cast<unsigned int*>(ix->vm[3].base);
  if (ix->keep_rows() && !ix->rows_on_host) ix->rows_x = reinterpret_cast<void*>(ix->vm[4].base);
  return RBK_OK;
}

void vm_free(rbk_index* ix) {
  for (VmRange& r : ix->vm) {
    vm_unmap_from(&r, 0);
    if (r.reserved) vmm_api().MemAddressFree(r.base, r.reserved);
    r = VmRange();
  }
}

// Reserves an empty range of at least `bytes` (whole granules) into *r.
rbk_status vm_reserve_range(const rbk_index* ix, size_t bytes, VmRange* r) {
  *r = VmRange();
  const size_t len = static_cast<size_t>(round_up(static_cast<int64_t>(bytes), static_cast<int64_t>(ix->vm_gran)));
  const CUresult res = vmm_api().MemAddressReserve(&r->base, len, 0, 0, 0);
  if (res != CUDA_SUCCESS) return cu_fail(res, "cuMemAddressReserve");
  r->reserved = len;
  return RBK_OK;
}

// Unmaps every chunk of r and frees its address range; the physical chunks are NOT released (another range maps them).
void vm_drop_mapping(VmRange* r) {
  const VmmApi& api = vmm_api();
  size_t off = 0;
  for (const VmRange::Chunk& c : r->chunks) {
    api.MemUnmap(r->base + off, c.bytes);
    off += c.bytes;
  }
  if (r->reserved) api.MemAddressFree(r->base, r->reserved);
  *r = VmRange();
}

// A second mapping of src's physical chunks, in the same order, on a new range of `bytes` (>= src.mapped): the same
// memory at another address, nothing copied.  On failure nothing is left reserved or mapped.
rbk_status vm_alias(const rbk_index* ix, const VmRange& src, size_t bytes, VmRange* out) {
  rbk_status st = vm_reserve_range(ix, bytes, out);
  if (st != RBK_OK) return st;
  const VmmApi& api = vmm_api();
  CUmemAccessDesc access;
  memset(&access, 0, sizeof access);
  access.location = vm_prop(ix->device).location;
  access.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  for (const VmRange::Chunk& c : src.chunks) {
    const CUdeviceptr at = out->base + out->mapped;
    CUresult res = api.MemMap(at, c.bytes, 0, c.handle, 0);
    if (res == CUDA_SUCCESS) {
      out->chunks.push_back(c);
      out->mapped += c.bytes;
      res = api.MemSetAccess(at, c.bytes, &access, 1);
    }
    if (res != CUDA_SUCCESS) {
      vm_drop_mapping(out);
      return cu_fail(res, "cuMemMap(index storage, new address range)");
    }
  }
  return RBK_OK;
}

// The pinned, mapped buffer of `bytes` that the exact rows of RBK_INDEX_ROWS_ON_HOST live in (one pointer under UVA).
rbk_status alloc_host_rows(size_t bytes, void** out) {
  void* r = nullptr;
  // not write-combined: the host reads these rows when the index grows
  cudaError_t e = cudaHostAlloc(&r, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
  if (e != cudaSuccess) return cuda_fail(e, "cudaHostAlloc(exact rows on the host)");
  void* dp = nullptr;
  if ((e = cudaHostGetDevicePointer(&dp, r, 0)) != cudaSuccess || dp != r) {
    cudaFreeHost(r);
    if (e != cudaSuccess) return cuda_fail(e, "cudaHostGetDevicePointer(exact rows on the host)");
    return fail(RBK_ECUDA, "pinned host rows are mapped at another device address (no unified addressing)");
  }
  *out = r;
  return RBK_OK;
}

// RBK_INDEX_ROWS_ON_HOST: a pinned buffer for `ncap` rows holding the first n_rows rows of the current one, which it
// replaces (peak: old + new in host RAM).  Synchronises the index stream first, so that every kernel that wrote or read
// the old rows has finished.
rbk_status realloc_host_rows(rbk_index* ix, int64_t ncap) {
  void* r = nullptr;
  rbk_status st = alloc_host_rows(static_cast<size_t>(ncap) * ix->x_row_bytes(), &r);
  if (st != RBK_OK) return st;
  cudaError_t e = cudaStreamSynchronize(ix->stream);
  if (e != cudaSuccess) {
    cudaFreeHost(r);
    return cuda_fail(e, "cudaStreamSynchronize");
  }
  if (ix->n_rows > 0) memcpy(r, ix->rows_x, static_cast<size_t>(ix->n_rows) * ix->x_row_bytes());
  if (ix->rows_x) cudaFreeHost(ix->rows_x);
  ix->rows_x = r;
  return RBK_OK;
}

// Grows the capacity in place: maps [cap, ncap) of every device buffer and initialises only that region.  Nothing is
// copied and no pointer moves.
rbk_status ensure_capacity(rbk_index* ix, int64_t need) {
  if (need <= ix->cap) return RBK_OK;
  if (need >= (1ll << 31) - 2 * kBlockN) return fail(RBK_EINVAL, "an index shard holds at most 2^31 rows");
  // whole 256-row tiles: the corpus tensor maps cover round_up(n_rows, 256) rows, so that no TMA box ever hangs over
  // the end of the tensor (the TMA unit zero-fills out-of-bounds rows one by one - see ensure_query_scratch)
  int64_t ncap = round_up(std::max<int64_t>(need, std::max<int64_t>(ix->cap * 2, 1024)), kBlockN);
  size_t old[rbk_index::kVmBuffers];
  for (int i = 0; i < rbk_index::kVmBuffers; ++i) old[i] = ix->vm[i].mapped;
  rbk_status st = vm_map_capacity(ix, ncap);
  if (st == RBK_ENOMEM && ncap > round_up(need, kBlockN)) {   // the doubled capacity cannot be backed: exactly `need`
    ncap = round_up(need, kBlockN);
    st = vm_map_capacity(ix, ncap);
  }
  if (st != RBK_OK) return st;
  if (ix->rows_on_host && (st = realloc_host_rows(ix, ncap)) != RBK_OK) {
    for (int i = 0; i < rbk_index::kVmBuffers; ++i) vm_unmap_from(&ix->vm[i], old[i]);
    return st;
  }
  cudaStream_t s = ix->stream;
  const int64_t cap = ix->cap;
  // rows not (yet) appended are read by the scan as part of the last tile (their 1/||c|| is NaN: they never match)
  CK(cudaMemsetAsync(ix->rows + static_cast<size_t>(cap) * ix->dpad, 0, static_cast<size_t>(ncap - cap) * ix->dpad * 2, s));
  CK(cudaMemsetAsync(ix->inv_norm + cap, 0xFF, static_cast<size_t>(inv_norm_len(ncap) - cap) * 4, s));   // all-ones = NaN
  CK(cudaMemsetAsync(ix->dead_bits + cap / 32, 0, static_cast<size_t>(ncap - cap) / 32 * 4, s));   // cap, ncap: x256
  ix->cap = ncap;
  return RBK_OK;
}

// src: host (is_device = false) or device rows of `elem` bytes (8 = f64, 4 = f32, 2 = bf16).
rbk_status append_rows(rbk_index* ix, const void* src, bool is_device, int elem, int64_t n, int64_t* first_out) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  if (n < 0 || (n > 0 && !src)) return fail(RBK_EINVAL, "bad rows argument");
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  if (first_out) *first_out = ix->n_rows;
  if (n == 0) return RBK_OK;
  // float32 exact rows take float64 sources only when every value fits: checked before anything is written
  rbk_status st = elem == 8 && ix->f32_rows()
                      ? check_f32_exact(ix, static_cast<const double*>(src), is_device, n * ix->dim)
                      : RBK_OK;
  if (st != RBK_OK) return st;
  st = ensure_capacity(ix, ix->n_rows + n);
  if (st != RBK_OK) return st;
  const int src_type = elem == 8 ? 0 : (elem == 4 ? 1 : 2);
  uint16_t* dst0 = ix->rows + static_cast<size_t>(ix->n_rows) * ix->dpad;
  unsigned char* dstx =
      ix->keep_rows() ? static_cast<unsigned char*>(ix->rows_x) + static_cast<size_t>(ix->n_rows) * ix->x_row_bytes()
                      : nullptr;
  if (is_device) {
    if (elem == 2 && ix->dpad == ix->dim && !ix->keep_rows()) {
      CK(cudaMemcpyAsync(dst0, src, static_cast<size_t>(n) * ix->dim * 2, cudaMemcpyDeviceToDevice, ix->stream));
    } else {
      CK(launch_convert_rows(src, src_type, n, ix->dim, ix->dpad, dst0, dstx, ix->x_elem, ix->stream, nullptr, nullptr,
                             nullptr, ix->scan_f16));
      ix->stats.kernel_launches++;
    }
  } else {
    const size_t row_bytes = static_cast<size_t>(ix->dim) * elem;
    const int64_t chunk_rows = std::max<int64_t>(1, std::min<int64_t>(n, (64ll << 20) / static_cast<int64_t>(row_bytes)));
    CK(ix->stage.ensure(static_cast<size_t>(chunk_rows) * row_bytes));
    for (int64_t r0 = 0; r0 < n; r0 += chunk_rows) {
      const int64_t nr = std::min<int64_t>(chunk_rows, n - r0);
      const unsigned char* hp = static_cast<const unsigned char*>(src) + static_cast<size_t>(r0) * row_bytes;
      CK(cudaMemcpyAsync(ix->stage.p, hp, static_cast<size_t>(nr) * row_bytes, cudaMemcpyHostToDevice, ix->stream));
      CK(launch_convert_rows(ix->stage.p, src_type, nr, ix->dim, ix->dpad, dst0 + static_cast<size_t>(r0) * ix->dpad,
                             dstx ? dstx + static_cast<size_t>(r0) * ix->x_row_bytes() : nullptr, ix->x_elem, ix->stream,
                             nullptr, nullptr, nullptr, ix->scan_f16));
      ix->stats.kernel_launches++;
      // the staging buffer is reused by the next chunk; pageable H2D copies are already
      // synchronous with respect to the host buffer, the kernel is ordered by the stream
    }
  }
  CK(launch_row_norms(ix->rows, ix->rows_x, ix->x_elem, ix->n_rows, n, ix->dim, ix->dpad, ix->inv_norm, ix->norm2,
                      ix->d_counter + 1, ix->stream, nullptr, nullptr, ix->scan_f16));
  ix->stats.kernel_launches += ix->keep_rows() ? 2 : 1;
  // Host sources: pageable H2D copies have consumed the caller's buffer when cudaMemcpyAsync returns and everything
  // after is stream-ordered, so an append costs no host round trip.  Device sources are read by the copy/convert
  // kernel itself, and page-locked host sources by a copy that really is asynchronous: the caller may free or reuse
  // either as soon as we return, so wait for those.
  if (is_device || host_source_is_pinned(src)) CK(cudaStreamSynchronize(ix->stream));
  ix->n_rows += n;
  ix->n_live += n;
  return RBK_OK;
}

int pick_kprime(const rbk_index* ix, int k_fetch) {
  if (ix->kprime_override > 0) return ix->kprime_override;
  int kp = static_cast<int>(round_up(k_fetch + ix->margin, 16));
  return std::min(kp, kMaxKPrime);
}

rbk_status refresh_corpus_tmap(rbk_index* ix) {
  const int64_t map_rows = round_up(ix->n_rows, kBlockN);   // whole tiles (<= cap): no out-of-bounds box rows
  if (ix->tmap_c_rows == map_rows) return RBK_OK;
  rbk_status st = encode_rows_tmap(&ix->tmap_c, ix->rows, map_rows, ix->dpad, kBlockN, ix->scan_f16);
  if (st != RBK_OK) return st;
  ix->tmap_c_rows = map_rows;
  return RBK_OK;
}

QueryBuffers query_buffers(rbk_index* ix, int q0) {
  QueryBuffers qb;
  qb.q_bf16 = ix->q_bf16.p + static_cast<size_t>(q0) * ix->dpad;
  qb.q_f64 = ix->q_f64.p + static_cast<size_t>(q0) * ix->dim;
  qb.q_norm2 = ix->q_norm2.p + q0;
  qb.q_inv_norm = ix->q_inv_norm.p + q0;
  qb.q_eps = ix->q_eps.p + q0;
  qb.thr_init = ix->thr_init.p + q0;
  return qb;
}

// ---- one scan launch per sub-batch of at most kMaxSubBatch queries, in every mode ----
// A launch's scratch is one buffer, ix->hist, split for a sub-batch of Bs queries as
//   hist [Bs][kHistBins] | maxbin [Bs] | gthr [Bs] | progress [sm_count + 8]
// and zeroed before every launch: by the prep kernel for the first sub-batch, by zero_scan_scratch for the others.
int progress_slots(const rbk_index* ix) { return ix->sm_count + 8; }
size_t scan_scratch_words(const rbk_index* ix, int Bs) {
  return static_cast<size_t>(Bs) * kHistBins + 2 * Bs + progress_slots(ix);
}

// The fields every scan mode shares, for the Bs queries from q0 on, against the rows from local row r0 on (a multiple
// of kBlockN, with a corpus map that starts there: rbk_index_similar_pairs_f64).
void fill_scan_params(rbk_index* ix, int q0, int Bs, int kprime, ScanParams* sp, int64_t r0 = 0) {
  const int64_t n_rows = ix->n_rows - r0;
  const int n_tiles = static_cast<int>((n_rows + kBlockN - 1) / kBlockN);
  const int QB = (Bs + kBlockM - 1) / kBlockM;
  sp->inv_norm_c = ix->inv_norm + r0;
  sp->thr_init = ix->thr_init.p + q0;
  sp->inv_norm_q = ix->q_inv_norm.p + q0;
  sp->hist = ix->hist.p;
  sp->maxbin = reinterpret_cast<int*>(ix->hist.p + static_cast<size_t>(Bs) * kHistBins);
  sp->gthr = reinterpret_cast<unsigned int*>(sp->maxbin + Bs);
  sp->progress = sp->maxbin + 2 * Bs;
  sp->n_rows = static_cast<int>(n_rows);
  sp->B = Bs;
  sp->kprime = kprime;
  sp->dpad = ix->dpad;
  sp->max_lead_tiles = ix->max_lead_tiles;
  sp->QB = QB;
  sp->R = std::max(1, std::min(ix->sm_count / QB, n_tiles));
  sp->n_tiles = n_tiles;
}

LargeScanParams large_scan_params(rbk_index* ix, int q0, int Bs, int k_fetch, int64_t r0 = 0) {
  LargeScanParams sp{};
  fill_scan_params(ix, q0, Bs, k_fetch, &sp, r0);
  sp.q_eps = ix->q_eps.p + q0;
  return sp;
}

cudaError_t zero_scan_scratch(rbk_index* ix, int Bs) {
  return cudaMemsetAsync(ix->hist.p, 0, sizeof(unsigned int) * scan_scratch_words(ix, Bs), ix->stream);
}

// The prep kernel for all B queries; it also zeroes the first sub-batch's scan scratch.
// min_each (nullable): each query's own min_score.
rbk_status prep_queries(rbk_index* ix, const void* d_q, int src_type, int B, double min_score, bool with_norm2,
                        const double* min_each = nullptr) {
  CK(launch_prep_queries(d_q, src_type, B, ix->dim, ix->dpad, min_score,
                         reinterpret_cast<const float*>(ix->d_counter + 1),
                         query_buffers(ix, 0), ix->stream, with_norm2, ix->hist.p, std::min(kMaxSubBatch, B),
                         progress_slots(ix), ix->scan_f16, min_each));
  ix->stats.kernel_launches++;
  return RBK_OK;
}

// Launches one filled sub-batch: its query map, then the scan kernel of kMode (0: the top-k' scan, P = ScanParams;
// kScanCount / kScanEmit: a large-k pass, P = LargeScanParams) inside a timing pair unless the stream is being captured.
// tmap_c (nullable): the corpus map, when it is not the index's own (rows from r0 on; see fill_scan_params).
template <int kMode, typename P>
rbk_status launch_sub_batch(rbk_index* ix, int q0, const P& sp, const CUtensorMap* tmap_c = nullptr) {
  if (!tmap_c) tmap_c = &ix->tmap_c;
  CUtensorMap tmap_q;
  const int q_rows = static_cast<int>(round_up(sp.B, kBlockM));   // whole query blocks: no out-of-bounds box rows
  // every row the map covers must lie inside the query buffer: the scan's TMA loads whole boxes
  if ((static_cast<size_t>(q0) + q_rows) * ix->dpad > ix->q_bf16.n)
    return fail(RBK_ECUDA, "scan launch at query " + std::to_string(q0) + " would read past the query buffer");
  rbk_status st = encode_rows_tmap(&tmap_q, ix->q_bf16.p + static_cast<size_t>(q0) * ix->dpad, q_rows, ix->dpad, kBlockM,
                                   ix->scan_f16);
  if (st != RBK_OK) return st;
  cudaEvent_t* tev = ix->capturing ? nullptr : next_scan_events(ix);
  if (tev) CK(cudaEventRecord(tev[0], ix->stream));
  if constexpr (kMode == 0)
    CK((ix->scan_f16 ? launch_scan_f16 : launch_scan)(tmap_q, *tmap_c, sp, ix->stream));
  else
    CK((ix->scan_f16 ? launch_scan_large_f16 : launch_scan_large)(tmap_q, *tmap_c, sp,
                                                                  static_cast<LargeScanMode>(kMode), ix->stream));
  if (tev) CK(cudaEventRecord(tev[1], ix->stream));
  ix->stats.last_ring_stages = kStages;
  ix->stats.scan_launches++;
  ix->stats.kernel_launches++;
  return RBK_OK;
}

// Results of a search over an empty index: -1 slots, zero counts, and NaN scores with the bits every other path
// writes (the quiet NaN 0x7FF8000000000000), so an empty index answers byte for byte as an empty group does.
rbk_status fill_empty_results(rbk_index* ix, int B, int k_fetch, long long* d_slots, double* d_scores, int* d_counts) {
  CK(cudaMemsetAsync(d_counts, 0, sizeof(int) * B, ix->stream));
  const int64_t n = static_cast<int64_t>(B) * k_fetch;
  if (n > 0) {
    empty_results_kernel<<<static_cast<unsigned>(std::min<int64_t>((n + 255) / 256, 1024)), 256, 0, ix->stream>>>(
        d_slots, d_scores, n);
    CK(cudaGetLastError());
  }
  return RBK_OK;
}

}  // namespace

// ---- shared with rbk_group.cu (declared in rbk_index_impl.h) ----
namespace rbk {
namespace impl {

rbk_status ensure_query_scratch(rbk_index* ix, int B, int elem) {
  CK(ix->q_raw.ensure(static_cast<size_t>(B) * ix->dim * elem));
  // rows padded to whole query blocks: the scan's TMA boxes are 128 query rows, and a box that hangs over the end of
  // the tensor is zero-FILLED by the TMA unit row by row, which is slow.  With the map covering whole blocks the pad
  // rows are ordinary (zeroed once here) memory; they only ever feed accumulator rows of queries that do not exist.
  // One more block of them lets a large-k search's query group start its map at any query.
  {
    const size_t want = static_cast<size_t>(round_up(B, kBlockM) + kBlockM) * ix->dpad;
    if (want > ix->q_bf16.n) {
      CK(ix->q_bf16.ensure(want));
      CK(cudaMemsetAsync(ix->q_bf16.p, 0, ix->q_bf16.n * sizeof(uint16_t), ix->stream));
    }
  }
  CK(ix->q_f64.ensure(static_cast<size_t>(B) * ix->dim));
  CK(ix->q_norm2.ensure(B));
  CK(ix->q_eps.ensure(B));
  CK(ix->q_inv_norm.ensure(B));
  CK(ix->thr_init.ensure(B));
  CK(ix->flags.ensure(B));
  CK(ix->cand.ensure(static_cast<size_t>(ix->sm_count) * kBlockM * kListCap));
  CK(ix->cand_cnt.ensure(static_cast<size_t>(ix->sm_count) * kBlockM));
  CK(ix->hist.ensure(scan_scratch_words(ix, kMaxSubBatch)));
  return RBK_OK;
}

rbk_status check_search_args(rbk_index* ix, int B, bool have_q, int query_dim, int k_fetch, double min_score,
                             int max_k) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  if (B < 0 || (B > 0 && !have_q)) return fail(RBK_EINVAL, "bad queries argument");
  if (k_fetch < 1 || k_fetch > max_k) return fail(RBK_EINVAL, "k_fetch must be in [1, " + std::to_string(max_k) + "]");
  if (query_dim != ix->dim) return fail(RBK_EDIM, "Vectors must have the same length");  // embedder.ts:170
  if (min_score != min_score) return fail(RBK_EINVAL, "min_score is NaN");
  return RBK_OK;
}

rbk_status check_each_args(rbk_index* ix, int B, bool have_q, int query_dim, const int32_t* k, const double* min_score,
                           int* K) {
  *K = 0;
  if (!ix) return fail(RBK_EINVAL, "null index");
  if (B < 0 || (B > 0 && !have_q)) return fail(RBK_EINVAL, "bad queries argument");
  if (B > 0 && (!k || !min_score)) return fail(RBK_EINVAL, "null k_fetch or min_score array");
  for (int b = 0; b < B; ++b) {
    if (k[b] < 1) return fail(RBK_EINVAL, "k_fetch[" + std::to_string(b) + "] must be >= 1");
    *K = std::max(*K, static_cast<int>(k[b]));
  }
  if (query_dim != ix->dim) return fail(RBK_EDIM, "Vectors must have the same length");  // embedder.ts:170
  for (int b = 0; b < B; ++b)
    if (min_score[b] != min_score[b]) return fail(RBK_EINVAL, "min_score[" + std::to_string(b) + "] is NaN");
  return RBK_OK;
}

rbk_status upload_cuts(rbk_index* ix, int B, const int32_t* k, const double* min_score, QueryCuts* out) {
  CK(ix->e_k.ensure(B));
  CK(ix->e_min.ensure(B));
  // pageable sources: both copies have read the caller's arrays when they return
  CK(cudaMemcpyAsync(ix->e_k.p, k, sizeof(int) * B, cudaMemcpyHostToDevice, ix->stream));
  CK(cudaMemcpyAsync(ix->e_min.p, min_score, sizeof(double) * B, cudaMemcpyHostToDevice, ix->stream));
  out->k = ix->e_k.p;
  out->min_score = ix->e_min.p;
  return RBK_OK;
}

rbk_status gather_queries(rbk_index* ix, const int64_t* rows, int B) {
  CK(ix->q_raw.ensure(static_cast<size_t>(B) * ix->dim * 8));
  CK(ix->sq_rows.ensure(B));
  CK(ix->sq_dead.ensure(1));
  CK(ix->h_sq_dead.ensure(1));
  // pageable source: the copy has read the caller's rows when it returns
  CK(cudaMemcpyAsync(ix->sq_rows.p, rows, sizeof(int64_t) * B, cudaMemcpyHostToDevice, ix->stream));
  CK(cudaMemsetAsync(ix->sq_dead.p, 0, sizeof(int), ix->stream));
  CK(launch_gather_rows(ix->rows, ix->rows_x, ix->x_elem, ix->dead_bits, ix->sq_rows.p, B, ix->dim, ix->dpad,
                        reinterpret_cast<double*>(ix->q_raw.p), ix->sq_dead.p, ix->stream));
  ix->stats.kernel_launches++;
  CK(cudaMemcpyAsync(ix->h_sq_dead.p, ix->sq_dead.p, sizeof(int), cudaMemcpyDeviceToHost, ix->stream));
  return RBK_OK;
}

rbk_status check_gathered(const rbk_index* ix) {
  if (ix->h_sq_dead.p[0] == 0) return RBK_OK;
  return fail(RBK_EINVAL, "query slot is tombstoned (" + std::to_string(ix->h_sq_dead.p[0]) + " of the batch)");
}

rbk_status check_mmr_args(rbk_index* ix, int B, bool have_q, int query_dim, const int32_t* k, const int32_t* fetch_k,
                          const double* lambda_mult, const double* min_score, const void* out_slots,
                          const void* out_scores, const void* out_counts, int* K) {
  *K = 0;
  if (!ix) return fail(RBK_EINVAL, "null index");
  if (B < 0 || (B > 0 && !have_q)) return fail(RBK_EINVAL, "bad queries argument");
  if (B > 0 && (!k || !fetch_k || !lambda_mult || !min_score))
    return fail(RBK_EINVAL, "null k, fetch_k, lambda_mult or min_score array");
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  for (int b = 0; b < B; ++b) {
    const std::string at = "[" + std::to_string(b) + "]";
    if (k[b] < 1) return fail(RBK_EINVAL, "k" + at + " must be >= 1");
    if (fetch_k[b] < k[b]) return fail(RBK_EINVAL, "fetch_k" + at + " must be >= k" + at);
    if (fetch_k[b] > RBK_MAX_K_FETCH_LARGE)
      return fail(RBK_EINVAL, "fetch_k" + at + " must be <= " + std::to_string(RBK_MAX_K_FETCH_LARGE));
    if (static_cast<int64_t>(fetch_k[b]) * ix->dim > RBK_MMR_MAX_FETCH_ELEMS)
      return fail(RBK_EINVAL, "fetch_k" + at + " * dim must be <= RBK_MMR_MAX_FETCH_ELEMS");
    *K = std::max(*K, static_cast<int>(k[b]));
  }
  if (query_dim != ix->dim) return fail(RBK_EDIM, "Vectors must have the same length");  // embedder.ts:170
  for (int b = 0; b < B; ++b) {
    if (min_score[b] != min_score[b]) return fail(RBK_EINVAL, "min_score[" + std::to_string(b) + "] is NaN");
    if (!(lambda_mult[b] >= 0.0 && lambda_mult[b] <= 1.0))
      return fail(RBK_EINVAL, "lambda_mult[" + std::to_string(b) + "] must be in [0, 1]");
  }
  return RBK_OK;
}

rbk_status mmr_select_locked(rbk_index* ix, int Bc, int F, const int64_t* c_slots, const double* c_scores,
                             const int32_t* c_counts, const int32_t* k, const double* lambda_mult, int K,
                             const MmrStage& stage, bool check_dead, int64_t* out_slots, double* out_scores,
                             int32_t* out_counts, float* ms_out) {
  std::vector<int64_t> cost(Bc);
  for (int b = 0; b < Bc; ++b) {
    cost[b] = static_cast<int64_t>(c_counts[b]) * ix->dim * 8;
    out_counts[b] = std::min(k[b], c_counts[b]);
  }
  // RBK_MMR_MAX_FETCH_ELEMS keeps every query's rows within the budget, so a group of one always fits
  for (const auto& gr : split_by_budget(cost)) {
    const int q0 = gr.first, Bg = gr.second - gr.first;
    // packed inputs: off i64 [Bg + 1] | slots i64 [M] | rel f64 [M] | lambda f64 [Bg] | k i32 [Bg]
    std::vector<int64_t> off(Bg + 1, 0);
    int max_m = 0;
    for (int b = 0; b < Bg; ++b) {
      off[b + 1] = off[b] + c_counts[q0 + b];
      max_m = std::max(max_m, static_cast<int>(c_counts[q0 + b]));
    }
    const int64_t M = off[Bg];
    const size_t o_slots = 8 * static_cast<size_t>(Bg + 1), o_rel = o_slots + 8 * M, o_lam = o_rel + 8 * M,
                 o_k = o_lam + 8 * static_cast<size_t>(Bg), bytes = o_k + 4 * static_cast<size_t>(Bg);
    std::vector<unsigned char> h(bytes);
    memcpy(h.data(), off.data(), o_slots);
    int64_t* h_slots = reinterpret_cast<int64_t*>(h.data() + o_slots);
    double* h_rel = reinterpret_cast<double*>(h.data() + o_rel);
    for (int b = 0; b < Bg; ++b) {
      memcpy(h_slots + off[b], c_slots + static_cast<size_t>(q0 + b) * F, 8 * static_cast<size_t>(c_counts[q0 + b]));
      memcpy(h_rel + off[b], c_scores + static_cast<size_t>(q0 + b) * F, 8 * static_cast<size_t>(c_counts[q0 + b]));
    }
    memcpy(h.data() + o_lam, lambda_mult + q0, 8 * static_cast<size_t>(Bg));
    memcpy(h.data() + o_k, k + q0, 4 * static_cast<size_t>(Bg));
    const size_t nk = static_cast<size_t>(Bg) * K;
    CK(ix->mm_in.ensure(bytes));
    CK(ix->mm_out.ensure(16 * nk));
    rbk_status st = stage.host(h_slots, static_cast<int>(M));
    if (st != RBK_OK) return st;
    CK(cudaEventRecord(ix->ev_start, ix->stream));
    if ((st = stage.device(static_cast<int>(M))) != RBK_OK) return st;
    // pageable source: the copy has read h when it returns
    CK(cudaMemcpyAsync(ix->mm_in.p, h.data(), bytes, cudaMemcpyHostToDevice, ix->stream));
    unsigned char* in = ix->mm_in.p;
    int64_t* d_slots = reinterpret_cast<int64_t*>(ix->mm_out.p);
    double* d_scores = reinterpret_cast<double*>(ix->mm_out.p + 8 * nk);
    CK(launch_mmr_select(reinterpret_cast<const double*>(ix->q_raw.p), ix->dim, reinterpret_cast<const int64_t*>(in),
                         reinterpret_cast<const int64_t*>(in + o_slots), reinterpret_cast<const double*>(in + o_rel),
                         reinterpret_cast<const int*>(in + o_k), reinterpret_cast<const double*>(in + o_lam), Bg,
                         max_m, K, d_slots, d_scores, ix->stream));
    ix->stats.kernel_launches++;
    CK(cudaEventRecord(ix->ev_stop, ix->stream));
    CK(cudaMemcpyAsync(out_slots + static_cast<size_t>(q0) * K, d_slots, 8 * nk, cudaMemcpyDeviceToHost, ix->stream));
    CK(cudaMemcpyAsync(out_scores + static_cast<size_t>(q0) * K, d_scores, 8 * nk, cudaMemcpyDeviceToHost,
                       ix->stream));
    CK(cudaStreamSynchronize(ix->stream));
    if (check_dead && M > 0 && ix->h_sq_dead.p[0] != 0)
      return fail(RBK_ECUDA, "MMR: " + std::to_string(ix->h_sq_dead.p[0]) + " candidate rows were tombstoned");
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ix->ev_start, ix->ev_stop));
    *ms_out += ms;
  }
  return RBK_OK;
}

}  // namespace impl
}  // namespace rbk

namespace {

// Launch the scan (+ optionally finalize) for every sub-batch.  d_q: device queries.  each: per-query cuts (k_fetch is
// then the largest k: it sets k' for the whole batch, and the row stride).
rbk_status run_scan(rbk_index* ix, const void* d_q, int src_type, int B, int k_fetch, double min_score,
                    long long* d_slots, double* d_scores, int* d_counts, int* d_flags, float* dbg,
                    const QueryCuts& each = QueryCuts()) {
  const int kprime = pick_kprime(ix, k_fetch);
  ix->stats.last_kprime = kprime;
  // normA is left to the finalize kernel
  rbk_status st = prep_queries(ix, d_q, src_type, B, min_score, /*with_norm2=*/d_counts == nullptr, each.min_score);
  if (st != RBK_OK) return st;
  if (ix->n_rows == 0) {
    // nothing to scan: finalize would read unwritten lists; emit empty results directly
    if (d_counts) {
      st = fill_empty_results(ix, B, k_fetch, d_slots, d_scores, d_counts);
      if (st != RBK_OK) return st;
      CK(cudaMemsetAsync(d_flags, 0, sizeof(int) * B, ix->stream));
    }
    return RBK_OK;
  }
  st = refresh_corpus_tmap(ix);
  if (st != RBK_OK) return st;
  for (int q0 = 0; q0 < B; q0 += kMaxSubBatch) {
    const int Bs = std::min(kMaxSubBatch, B - q0);
    if (q0 > 0) CK(zero_scan_scratch(ix, Bs));
    ScanParams sp;
    fill_scan_params(ix, q0, Bs, kprime, &sp);
    sp.cand = ix->cand.p;
    sp.cand_cnt = ix->cand_cnt.p;
    sp.dbg_scores = dbg ? dbg + static_cast<size_t>(q0) * ix->n_rows : nullptr;
    st = launch_sub_batch<0>(ix, q0, sp);
    if (st != RBK_OK) return st;
    if (d_counts) {
      FinalizeParams fp;
      fp.cand = ix->cand.p;
      fp.cand_cnt = ix->cand_cnt.p;
      fp.QB = sp.QB;
      fp.R = sp.R;
      fp.kprime = kprime;
      fp.k_fetch = k_fetch;
      fp.B = Bs;
      fp.d = ix->dim;
      fp.dpad = ix->dpad;
      fp.q0 = q0;
      fp.block_m = kBlockM;
      fp.min_score = min_score;
      fp.rows = ix->rows;
      fp.rows_x = ix->rows_x;
      fp.row_norm2 = ix->norm2;
      fp.n_rows = ix->n_rows;
      fp.slot = ix->slot;
      fp.q = query_buffers(ix, q0);
      fp.out_slots = d_slots + static_cast<size_t>(q0) * k_fetch;
      fp.out_scores = d_scores + static_cast<size_t>(q0) * k_fetch;
      fp.out_counts = d_counts + q0;
      fp.flags = d_flags + q0;
      fp.k_each = each.k ? each.k + q0 : nullptr;
      fp.min_each = each.min_score ? each.min_score + q0 : nullptr;
      CK(launch_finalize(fp, ix->rows_on_host, ix->x_elem, ix->stream));
      ix->stats.kernel_launches++;
    }
  }
  return RBK_OK;
}

rbk_status run_fallback(rbk_index* ix, const std::vector<int>& fails, int k_fetch, double min_score,
                        long long* d_slots, double* d_scores, int* d_counts, const QueryCuts& each = QueryCuts()) {
  const int nf = static_cast<int>(fails.size());
  const int nb = std::max(1, std::min<int>(ix->sm_count * 2, static_cast<int>((ix->n_rows + 255) / 256)));
  CK(ix->fail_list.ensure(nf));
  CK(ix->part_scores.ensure(static_cast<size_t>(nf) * nb * k_fetch));
  CK(ix->part_rows.ensure(static_cast<size_t>(nf) * nb * k_fetch));
  CK(ix->part_cnt.ensure(static_cast<size_t>(nf) * nb));
  CK(cudaMemcpyAsync(ix->fail_list.p, fails.data(), sizeof(int) * nf, cudaMemcpyHostToDevice, ix->stream));
  ExactParams ep;
  ep.fail_list = ix->fail_list.p;
  ep.n_fail = nf;
  ep.d = ix->dim;
  ep.dpad = ix->dpad;
  ep.k_fetch = k_fetch;
  ep.min_score = min_score;
  ep.rows = ix->rows;
  ep.rows_x = ix->rows_x;
  ep.row_norm2 = ix->norm2;
  ep.dead_bits = ix->dead_bits;
  ep.n_rows = ix->n_rows;
  ep.slot = ix->slot;
  ep.q_f64 = ix->q_f64.p;
  ep.q_norm2 = ix->q_norm2.p;
  ep.part_scores = ix->part_scores.p;
  ep.part_rows = ix->part_rows.p;
  ep.part_cnt = ix->part_cnt.p;
  ep.n_blocks = nb;
  ep.out_slots = d_slots;
  ep.out_scores = d_scores;
  ep.out_counts = d_counts;
  ep.k_each = each.k;
  ep.min_each = each.min_score;
  CK(launch_exact_fallback(ep, ix->x_elem, ix->stream));
  // pageable source: the copy above has completed its host read before returning
  ix->stats.kernel_launches += 2;
  ix->stats.fallback_queries += nf;
  return RBK_OK;
}

}  // namespace

namespace rbk {
namespace impl {
// Enqueue-only search of device-resident queries (caller holds the lock).  No host synchronisation: the
// exactness flags land in d_flags and are the caller's to check (rbk_index_search_device_async, rbk_group.cu).
rbk_status enqueue_search(rbk_index* ix, const void* d_q, int src_type, int B, int k_fetch, double min_score,
                          long long* d_slots, double* d_scores, int* d_counts, int* d_flags, const QueryCuts& each) {
  ix->stats.searches++;
  ix->stats.queries += B;
  return run_scan(ix, d_q, src_type, B, k_fetch, min_score, d_slots, d_scores, d_counts, d_flags, nullptr, each);
}

rbk_status large_count(rbk_index* ix, const void* d_q, int B, int k_eff, double min_score, const QueryCuts& each) {
  ix->stats.searches++;
  ix->stats.queries += B;
  ix->stats.last_kprime = k_eff;
  CK(ix->lg_theta.ensure(B));
  CK(ix->lg_cap.ensure(B));
  CK(ix->lg_cnt.ensure(B));
  CK(ix->lg_off.ensure(B));
  CK(ix->lg_err.ensure(1));
  CK(ix->h_lcap.ensure(B));
  CK(ix->h_loff.ensure(B));
  CK(ix->h_lerr.ensure(1));
  // normA is computed here: the re-rank has no spare thread to walk the chain beside its candidates
  rbk_status st = prep_queries(ix, d_q, 0, B, min_score, /*with_norm2=*/true, each.min_score);
  if (st != RBK_OK) return st;
  if (ix->n_rows == 0) {
    memset(ix->h_lcap.p, 0, sizeof(int) * B);
    return RBK_OK;
  }
  st = refresh_corpus_tmap(ix);
  if (st != RBK_OK) return st;
  for (int q0 = 0; q0 < B; q0 += kMaxSubBatch) {
    const int Bs = std::min(kMaxSubBatch, B - q0);
    if (q0 > 0) CK(zero_scan_scratch(ix, Bs));
    const LargeScanParams sp = large_scan_params(ix, q0, Bs, k_eff);
    st = launch_sub_batch<kScanCount>(ix, q0, sp);
    if (st != RBK_OK) return st;
    CK(launch_large_select(sp.hist, sp.thr_init, sp.inv_norm_q, sp.q_eps, Bs, k_eff, static_cast<int>(ix->n_rows),
                           ix->lg_theta.p + q0, ix->lg_cap.p + q0, ix->stream, each.k ? each.k + q0 : nullptr));
    ix->stats.kernel_launches++;
  }
  CK(cudaMemcpyAsync(ix->h_lcap.p, ix->lg_cap.p, sizeof(int) * B, cudaMemcpyDeviceToHost, ix->stream));
  return RBK_OK;
}

rbk_status large_check(rbk_index* ix) {
  if (ix->h_lerr.p[0] == 0) return RBK_OK;
  return fail(RBK_ECUDA, "large-k search: the emit scan found more rows than the count scan bounded for " +
                             std::to_string(ix->h_lerr.p[0]) + " queries (the answer is not proven exact)");
}

std::vector<std::pair<int, int>> split_by_budget(const std::vector<int64_t>& cost) {
  std::vector<std::pair<int, int>> groups;
  const int B = static_cast<int>(cost.size());
  int q0 = 0;
  int64_t used = 0;
  for (int b = 0; b < B; ++b) {
    if (b > q0 && used + cost[b] > kLargeBudget) {
      groups.emplace_back(q0, b);
      q0 = b;
      used = 0;
    }
    used += cost[b];
  }
  if (B > q0) groups.emplace_back(q0, B);
  return groups;
}

static int64_t sort_tiles(int cap) { return (cap + kSortTile - 1) / kSortTile; }

rbk_status large_prepare(rbk_index* ix, int B, bool sorted, const std::vector<std::pair<int, int>>& groups) {
  if (sorted) {
    CK(ix->h_utoff.ensure(B));
    CK(ix->ub_toff.ensure(B));
  }
  int64_t max_cand = 1, max_tiles = 1;
  for (const auto& gr : groups) {
    int64_t cand = 0, tiles = 0;
    for (int b = gr.first; b < gr.second; ++b) {
      ix->h_loff.p[b] = cand;
      cand += ix->h_lcap.p[b];
      if (sorted) {
        ix->h_utoff.p[b] = static_cast<int>(tiles);
        tiles += sort_tiles(ix->h_lcap.p[b]);
      }
    }
    max_cand = std::max(max_cand, cand);
    max_tiles = std::max(max_tiles, tiles);
  }
  CK(ix->lg_rows.ensure(static_cast<size_t>(max_cand)));
  CK(ix->lg_scores.ensure(static_cast<size_t>(max_cand)));
  CK(cudaMemcpyAsync(ix->lg_off.p, ix->h_loff.p, sizeof(long long) * B, cudaMemcpyHostToDevice, ix->stream));
  if (sorted) {
    CK(ix->ub_rows.ensure(static_cast<size_t>(max_cand)));
    CK(ix->ub_scores.ensure(static_cast<size_t>(max_cand)));
    CK(ix->ub_len.ensure(static_cast<size_t>(2 * max_tiles)));
    CK(cudaMemcpyAsync(ix->ub_toff.p, ix->h_utoff.p, sizeof(int) * B, cudaMemcpyHostToDevice, ix->stream));
  }
  CK(cudaMemsetAsync(ix->lg_cnt.p, 0, sizeof(int) * B, ix->stream));
  CK(cudaMemsetAsync(ix->lg_err.p, 0, sizeof(int), ix->stream));
  return RBK_OK;
}

rbk_status large_emit(rbk_index* ix, int q0, int q1, bool sorted, int k_eff, double min_score, long long* d_slots,
                      double* d_scores, int* d_counts, const QueryCuts& each) {
  if (ix->n_rows == 0) return fill_empty_results(ix, q1 - q0, k_eff, d_slots, d_scores, d_counts);
  int64_t group_tiles = 0;
  if (sorted)
    for (int b = q0; b < q1; ++b) group_tiles += sort_tiles(ix->h_lcap.p[b]);
  for (int s0 = q0; s0 < q1; s0 += kMaxSubBatch) {
    const int Bs = std::min(kMaxSubBatch, q1 - s0);
    LargeScanParams sp = large_scan_params(ix, s0, Bs, k_eff);
    sp.thr_init = ix->lg_theta.p + s0;   // theta_q of the count pass
    sp.emit_off = ix->lg_off.p + s0;
    sp.emit_cap = ix->lg_cap.p + s0;
    sp.emit_cnt = ix->lg_cnt.p + s0;
    sp.emit_rows = ix->lg_rows.p;
    CK(cudaMemsetAsync(sp.progress, 0, sizeof(int) * progress_slots(ix), ix->stream));
    rbk_status st = launch_sub_batch<kScanEmit>(ix, s0, sp);
    if (st != RBK_OK) return st;
    // a query whose bound proves nothing has C_q = n_rows (large_select); only then is there anything to emit
    if (std::find(ix->h_lcap.p + s0, ix->h_lcap.p + s0 + Bs, static_cast<int>(ix->n_rows)) != ix->h_lcap.p + s0 + Bs) {
      CK(launch_large_emit_all(ix->q_eps.p + s0, ix->dead_bits, ix->n_rows, Bs, sp.emit_off, sp.emit_cnt,
                               ix->lg_rows.p, ix->stream));
      ix->stats.kernel_launches++;
    }
    LargeRerankParams rp;
    rp.B = Bs;
    rp.d = ix->dim;
    rp.dpad = ix->dpad;
    rp.k_fetch = k_eff;
    rp.min_score = min_score;
    rp.rows = ix->rows;
    rp.rows_x = ix->rows_x;
    rp.row_norm2 = ix->norm2;
    rp.slot = ix->slot;
    rp.q_f64 = ix->q_f64.p + static_cast<size_t>(s0) * ix->dim;
    rp.q_norm2 = ix->q_norm2.p + s0;
    rp.emit_off = sp.emit_off;
    rp.emit_cap = sp.emit_cap;
    rp.emit_cnt = sp.emit_cnt;
    rp.emit_rows = ix->lg_rows.p;
    rp.cand_scores = ix->lg_scores.p;
    rp.out_slots = d_slots + static_cast<size_t>(s0 - q0) * k_eff;
    rp.out_scores = d_scores + static_cast<size_t>(s0 - q0) * k_eff;
    rp.out_counts = d_counts + (s0 - q0);
    rp.overflow = ix->lg_err.p;
    rp.k_each = each.k ? each.k + s0 : nullptr;
    rp.min_each = each.min_score ? each.min_score + s0 : nullptr;
    const int max_cap = *std::max_element(ix->h_lcap.p + s0, ix->h_lcap.p + s0 + Bs);
    SegSortScratch ss;
    if (sorted) {
      ss.tile_off = ix->ub_toff.p + s0;
      ss.scores = ix->ub_scores.p;
      ss.rows = ix->ub_rows.p;
      ss.len[0] = ix->ub_len.p;
      ss.len[1] = ix->ub_len.p + group_tiles;
      ss.max_tiles = static_cast<int>(sort_tiles(max_cap));
    }
    int launches = 0;
    CK(launch_large_rerank(rp, sorted ? &ss : nullptr, max_cap, ix->rows_on_host, ix->x_elem, ix->stream, &launches));
    ix->stats.kernel_launches += launches;
  }
  return RBK_OK;
}

rbk_status large_finish(rbk_index* ix) {
  CK(cudaMemcpyAsync(ix->h_lerr.p, ix->lg_err.p, sizeof(int), cudaMemcpyDeviceToHost, ix->stream));
  return RBK_OK;
}

int64_t first_row_at(const SlotLayout& s, int64_t a) {
  if (s.block == 0) return std::max<int64_t>(0, a - s.base);
  const int64_t blk = a / s.block, cycle = blk / s.G, pos = blk % s.G;
  if (pos == s.g) return cycle * s.block + a % s.block;
  return (pos < s.g ? cycle : cycle + 1) * s.block;   // the first row of this member's next block
}

rbk_status pairs_count(rbk_index* ix, int Q, int64_t a0, double min_score) {
  CK(ix->lg_theta.ensure(Q));
  CK(ix->lg_cap.ensure(Q));
  CK(ix->lg_cnt.ensure(Q));
  CK(ix->lg_off.ensure(Q));
  CK(ix->lg_err.ensure(1));
  CK(ix->h_lcap.ensure(Q));
  CK(ix->h_loff.ensure(Q));
  CK(ix->h_lerr.ensure(1));
  CK(ix->pr_cnt.ensure(Q));
  CK(ix->pr_off.ensure(Q));
  CK(ix->h_pcnt.ensure(Q));
  rbk_status st = prep_queries(ix, ix->q_raw.p, 0, Q, min_score, /*with_norm2=*/true);
  if (st != RBK_OK) return st;
  const int64_t first = first_row_at(ix->slot, a0);
  if (first >= ix->n_rows) {   // no row of this index can pair with the chunk
    ix->pr_rows = 0;
    memset(ix->h_lcap.p, 0, sizeof(int) * Q);
    return RBK_OK;
  }
  // the triangle: the scans read the rows from the chunk's first slot on, from a map that starts at the tile holding it
  ix->pr_r0 = first / kBlockN * kBlockN;
  ix->pr_rows = ix->n_rows - ix->pr_r0;
  st = encode_rows_tmap(&ix->pr_tmap, ix->rows + static_cast<size_t>(ix->pr_r0) * ix->dpad,
                        round_up(ix->n_rows, kBlockN) - ix->pr_r0, ix->dpad, kBlockN, ix->scan_f16);
  if (st != RBK_OK) return st;
  // k = INT32_MAX: the count pass never raises its threshold above min_score's, and the select keeps it (theta_q from
  // min_score and the query's bound alone, C_q every row counted at or above it)
  const LargeScanParams sp = large_scan_params(ix, 0, Q, INT32_MAX, ix->pr_r0);
  st = launch_sub_batch<kScanCount>(ix, 0, sp, &ix->pr_tmap);
  if (st != RBK_OK) return st;
  CK(launch_large_select(sp.hist, sp.thr_init, sp.inv_norm_q, sp.q_eps, Q, INT32_MAX, static_cast<int>(ix->pr_rows),
                         ix->lg_theta.p, ix->lg_cap.p, ix->stream));
  ix->stats.kernel_launches++;
  CK(cudaMemcpyAsync(ix->h_lcap.p, ix->lg_cap.p, sizeof(int) * Q, cudaMemcpyDeviceToHost, ix->stream));
  return RBK_OK;
}

rbk_status pairs_emit(rbk_index* ix, int q0, int q1, int64_t a0, double min_score) {
  const int Bs = q1 - q0;
  if (ix->pr_rows == 0) {
    memset(ix->h_pcnt.p, 0, sizeof(int) * Bs);
    ix->h_lerr.p[0] = 0;
    return RBK_OK;
  }
  const int64_t r0 = ix->pr_r0;
  int64_t cand = 0, group_tiles = 0;
  for (int b = q0; b < q1; ++b) {
    cand += ix->h_lcap.p[b];
    group_tiles += sort_tiles(ix->h_lcap.p[b]);
  }
  CK(ix->pr_b.ensure(static_cast<size_t>(std::max<int64_t>(cand, 1))));
  CK(ix->pr_s.ensure(static_cast<size_t>(std::max<int64_t>(cand, 1))));
  LargeScanParams sp = large_scan_params(ix, q0, Bs, INT32_MAX, r0);
  sp.thr_init = ix->lg_theta.p + q0;
  sp.emit_off = ix->lg_off.p + q0;
  sp.emit_cap = ix->lg_cap.p + q0;
  sp.emit_cnt = ix->lg_cnt.p + q0;
  sp.emit_rows = ix->lg_rows.p;
  CK(cudaMemsetAsync(sp.progress, 0, sizeof(int) * progress_slots(ix), ix->stream));
  rbk_status st = launch_sub_batch<kScanEmit>(ix, q0, sp, &ix->pr_tmap);
  if (st != RBK_OK) return st;
  if (std::find(ix->h_lcap.p + q0, ix->h_lcap.p + q1, static_cast<int>(ix->pr_rows)) != ix->h_lcap.p + q1) {
    CK(launch_large_emit_all(ix->q_eps.p + q0, ix->dead_bits + r0 / 32, ix->pr_rows, Bs, sp.emit_off, sp.emit_cnt,
                             ix->lg_rows.p, ix->stream));
    ix->stats.kernel_launches++;
  }
  LargeRerankParams rp{};
  rp.B = Bs;
  rp.d = ix->dim;
  rp.dpad = ix->dpad;
  rp.min_score = min_score;
  rp.rows = ix->rows + static_cast<size_t>(r0) * ix->dpad;
  rp.rows_x = ix->rows_x ? static_cast<const char*>(ix->rows_x) + static_cast<size_t>(r0) * ix->x_row_bytes() : nullptr;
  rp.row_norm2 = ix->norm2 + r0;
  rp.slot = ix->slot;
  rp.q_f64 = ix->q_f64.p + static_cast<size_t>(q0) * ix->dim;
  rp.q_norm2 = ix->q_norm2.p + q0;
  rp.emit_off = sp.emit_off;
  rp.emit_cap = sp.emit_cap;
  rp.emit_cnt = sp.emit_cnt;
  rp.emit_rows = ix->lg_rows.p;
  rp.cand_scores = ix->lg_scores.p;
  rp.overflow = ix->lg_err.p;
  const int max_cap = *std::max_element(ix->h_lcap.p + q0, ix->h_lcap.p + q1);
  SegSortScratch ss;
  ss.tile_off = ix->ub_toff.p + q0;
  ss.scores = ix->ub_scores.p;
  ss.rows = ix->ub_rows.p;
  ss.len[0] = ix->ub_len.p;
  ss.len[1] = ix->ub_len.p + group_tiles;
  ss.max_tiles = static_cast<int>(sort_tiles(max_cap));
  PairsParams pp;
  pp.a0 = a0 + q0;
  pp.r0 = r0;
  pp.counts = ix->pr_cnt.p;
  pp.offsets = ix->pr_off.p;
  pp.out_b = ix->pr_b.p;
  pp.out_scores = ix->pr_s.p;
  int launches = 0;
  CK(launch_pairs_rerank(rp, ss, max_cap, ix->rows_on_host, ix->x_elem, pp, ix->stream, &launches));
  ix->stats.kernel_launches += launches;
  CK(cudaMemcpyAsync(ix->h_pcnt.p, ix->pr_cnt.p, sizeof(int) * Bs, cudaMemcpyDeviceToHost, ix->stream));
  return large_finish(ix);
}

rbk_status pairs_fetch(rbk_index* ix, int64_t n) {
  if (n == 0) return RBK_OK;
  CK(ix->h_block.ensure(static_cast<size_t>(n) * 16));
  CK(cudaMemcpyAsync(ix->h_block.p, ix->pr_b.p, sizeof(long long) * n, cudaMemcpyDeviceToHost, ix->stream));
  CK(cudaMemcpyAsync(ix->h_block.p + n * 8, ix->pr_s.p, sizeof(double) * n, cudaMemcpyDeviceToHost, ix->stream));
  return RBK_OK;
}

}  // namespace impl
}  // namespace rbk

namespace {

void drop_graph(rbk_index* ix) {
  if (ix->graph_exec) cudaGraphExecDestroy(ix->graph_exec);
  ix->graph_exec = nullptr;
}

// Every grow-only scratch buffer (each is re-grown on demand by the next call that needs it) and the captured graph,
// which bakes in their pointers.  The stream must be idle.
void release_scratch(rbk_index* ix) {
  drop_graph(ix);
  ix->stage.release();
  ix->d_slots.release();
  ix->cp_map.release();
  ix->cp_scan.release();
  ix->q_raw.release();
  ix->q_bf16.release();
  ix->q_f64.release();
  ix->q_norm2.release();
  ix->q_eps.release();
  ix->q_inv_norm.release();
  ix->thr_init.release();
  ix->cand.release();
  ix->cand_cnt.release();
  ix->hist.release();
  ix->flags.release();
  ix->fail_list.release();
  ix->part_rows.release();
  ix->part_cnt.release();
  ix->o_scores.release();
  ix->part_scores.release();
  ix->dbg.release();
  ix->lg_theta.release();
  ix->lg_cap.release();
  ix->lg_cnt.release();
  ix->lg_rows.release();
  ix->lg_err.release();
  ix->lg_off.release();
  ix->lg_scores.release();
  ix->h_lcap.release();
  ix->h_lerr.release();
  ix->h_loff.release();
  ix->ub_toff.release();
  ix->ub_rows.release();
  ix->ub_len.release();
  ix->ub_scores.release();
  ix->h_utoff.release();
  ix->o_block.release();
  ix->h_block.release();
  ix->h_flags.release();
  ix->e_k.release();
  ix->e_min.release();
  ix->sq_rows.release();
  ix->sq_dead.release();
  ix->h_sq_dead.release();
  ix->mm_in.release();
  ix->mm_out.release();
  ix->h_q.release();
}

// Small-batch fast path of search_core (caller holds the lock; scratch, o_block and h_block are allocated): replay
// - or first capture - the graph of one whole search.  *done = true: results and flags are in h_block and every
// query is proven exact.  *done = false: something needs the general path (a query's proof failed), which the
// caller then runs from scratch.
rbk_status search_graph(rbk_index* ix, const void* q_host, int elem, int B, int k_fetch, double min_score,
                        const ResultBlock& L, bool* done) {
  *done = false;
  const size_t q_bytes = static_cast<size_t>(B) * ix->dim * elem;
  CK(ix->h_q.ensure(q_bytes));
  rbk_index::GraphKey key;
  memset(&key, 0, sizeof key);   // compared with memcmp: padding must be defined
  const void* ptrs[20] = {ix->rows, ix->inv_norm, ix->norm2, ix->rows_x, ix->dead_bits, ix->d_counter, ix->q_raw.p,
                          ix->q_bf16.p, ix->q_f64.p, ix->q_norm2.p, ix->q_eps.p, ix->q_inv_norm.p, ix->thr_init.p,
                          ix->cand.p, ix->cand_cnt.p, ix->hist.p, ix->o_block.p, ix->h_block.p, ix->h_q.p, nullptr};
  memcpy(key.ptr, ptrs, sizeof ptrs);
  key.n_rows = ix->n_rows;
  key.min_score = min_score;
  key.B = B;
  key.k_fetch = k_fetch;
  key.elem = elem;
  key.margin = ix->margin;
  key.slot = ix->slot;
  key.stream = ix->stream;
  unsigned char* base = ix->o_block.p;
  if (!ix->graph_exec || memcmp(&key, &ix->graph_key, sizeof key) != 0) {
    drop_graph(ix);
    cudaGraph_t graph = nullptr;
    CK(cudaStreamBeginCapture(ix->stream, cudaStreamCaptureModeThreadLocal));
    ix->capturing = true;
    cudaError_t e = cudaMemcpyAsync(ix->q_raw.p, ix->h_q.p, q_bytes, cudaMemcpyHostToDevice, ix->stream);
    rbk_status st = RBK_OK;
    if (e == cudaSuccess)
      st = run_scan(ix, ix->q_raw.p, elem == 8 ? 0 : 1, B, k_fetch, min_score, L.slots(base), L.scores(base),
                    L.counts(base), L.flags(base), nullptr);
    if (e == cudaSuccess && st == RBK_OK)
      e = cudaMemcpyAsync(ix->h_block.p, base, L.bytes, cudaMemcpyDeviceToHost, ix->stream);
    ix->capturing = false;
    const cudaError_t e2 = cudaStreamEndCapture(ix->stream, &graph);   // always leave capture mode
    if (st != RBK_OK) {
      if (graph) cudaGraphDestroy(graph);
      return st;
    }
    if (e != cudaSuccess || e2 != cudaSuccess || !graph) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      ix->use_graph = false;   // capture not possible here (e.g. the caller's stream is itself capturing): general
      return RBK_OK;           // path from now on, no retry per search
    }
    e = cudaGraphInstantiate(&ix->graph_exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) {
      ix->graph_exec = nullptr;
      cudaGetLastError();
      ix->use_graph = false;
      return RBK_OK;
    }
    memcpy(&ix->graph_key, &key, sizeof key);
  }
  memcpy(ix->h_q.p, q_host, q_bytes);
  CK(cudaEventRecord(ix->ev_start, ix->stream));
  CK(cudaGraphLaunch(ix->graph_exec, ix->stream));
  CK(cudaEventRecord(ix->ev_stop, ix->stream));
  CK(cudaStreamSynchronize(ix->stream));   // the one host round trip
  ix->stats.searches++;
  ix->stats.queries += B;
  ix->stats.scan_launches++;
  ix->stats.kernel_launches += 3;           // prep, scan, finalize (inside the graph)
  ix->stats.graph_replays++;
  const int* h_flags = L.flags(ix->h_block.p);
  for (int b = 0; b < B; ++b)
    if (h_flags[b]) return RBK_OK;          // a proof failed: the general path re-answers the batch
  float total = 0.f;
  cudaEventElapsedTime(&total, ix->ev_start, ix->ev_stop);
  ix->stats.last_total_ms = total;
  *done = true;
  return RBK_OK;
}

// Device-time frame of a synchronous search: begin() records the start event before its first work, every host
// round trip records the stop event and waits, and after the last one finish() takes the time of the whole search
// and of its scans.
struct TimedSearch {
  rbk_index* ix;
  double scan_ms0 = 0.0;
  rbk_status begin() {
    resolve_scan_events(ix, false);
    scan_ms0 = ix->stats.scan_ms_total;
    CK(cudaEventRecord(ix->ev_start, ix->stream));
    return RBK_OK;
  }
  rbk_status round_trip() {
    CK(cudaEventRecord(ix->ev_stop, ix->stream));
    CK(cudaStreamSynchronize(ix->stream));
    return RBK_OK;
  }
  void finish(float* ms_out) {
    float total = 0.f;
    cudaEventElapsedTime(&total, ix->ev_start, ix->ev_stop);
    resolve_scan_events(ix, true);   // the stream is idle: every pair is final
    ix->stats.last_total_ms = total;
    ix->stats.last_scan_ms = static_cast<float>(ix->stats.scan_ms_total - scan_ms0);
    if (ms_out) *ms_out = total;
  }
};

// Where a synchronous search's queries come from, exactly one of: a host array (`host`, of the search's elem bytes
// per element), queries already on the device (`dev`), or local rows of the index whose stored values are the queries
// (`rows`, host [B]: rbk_index_search_slots_f64).  The H2D or the gather into q_raw is the search's first timed work.
struct QuerySource {
  const void* host = nullptr;
  const void* dev = nullptr;
  const int64_t* rows = nullptr;
};

rbk_status load_queries(rbk_index* ix, const QuerySource& q, int B, int elem, const void** d_q) {
  *d_q = q.dev;
  if (q.rows) {
    rbk_status st = gather_queries(ix, q.rows, B);
    if (st != RBK_OK) return st;
    *d_q = ix->q_raw.p;
  } else if (q.host) {
    CK(cudaMemcpyAsync(ix->q_raw.p, q.host, static_cast<size_t>(B) * ix->dim * elem, cudaMemcpyHostToDevice,
                       ix->stream));
    *d_q = ix->q_raw.p;
  }
  return RBK_OK;
}

// Whole search, synchronous (caller holds the lock, device current, arguments checked).  Host outputs (out_*) may be
// null (device-output variant); device outputs may be null (host variant uses index scratch).  k_each / min_each (host
// [B], nullable; checked by the caller): a search_each call's cut and threshold per query, k_fetch their largest k; such
// a call never replays the captured graph, nor does a search of gathered rows.
rbk_status search_locked(rbk_index* ix, const QuerySource& q, int elem, int B, int k_fetch, double min_score,
                         long long* d_slots, double* d_scores, int* d_counts, int64_t* out_slots, double* out_scores,
                         int32_t* out_counts, float* ms_out, const int32_t* k_each = nullptr,
                         const double* min_each = nullptr) {
  rbk_status st;
  if (ms_out) *ms_out = 0.f;
  if (B == 0) {
    ix->stats.searches++;
    return RBK_OK;
  }
  st = ensure_query_scratch(ix, B, elem);
  if (st != RBK_OK) return st;
  // Host-output calls use ONE packed device block mirrored by one pinned host block, so results and exactness flags
  // come back in a single D2H copy.
  const ResultBlock L(B, k_fetch);
  const bool packed = d_slots == nullptr;
  int* d_flags = ix->flags.p;
  const int* h_flags = nullptr;
  if (packed) {
    CK(ix->o_block.ensure(L.bytes));
    CK(ix->h_block.ensure(L.bytes));
    d_slots = L.slots(ix->o_block.p);
    d_scores = L.scores(ix->o_block.p);
    d_counts = L.counts(ix->o_block.p);
    d_flags = L.flags(ix->o_block.p);
    h_flags = L.flags(ix->h_block.p);
  } else {
    CK(ix->h_flags.ensure(B));
    h_flags = ix->h_flags.p;
  }
  QueryCuts each;
  if (k_each) {
    st = upload_cuts(ix, B, k_each, min_each, &each);
    if (st != RBK_OK) return st;
  }
  if (packed && q.host && B <= kBlockM && ix->n_rows > 0 && ix->use_graph && !k_each) {
    bool done = false;
    st = search_graph(ix, q.host, elem, B, k_fetch, min_score, L, &done);
    if (st != RBK_OK) return st;
    if (done) {
      if (ms_out) *ms_out = ix->stats.last_total_ms;
      L.unpack(ix->h_block.p, out_slots, out_scores, out_counts);
      return RBK_OK;
    }
  }
  TimedSearch ts{ix};
  st = ts.begin();
  if (st != RBK_OK) return st;
  const void* d_q = nullptr;
  if ((st = load_queries(ix, q, B, elem, &d_q)) != RBK_OK) return st;
  const int src_type = elem == 8 ? 0 : 1;
  st = enqueue_search(ix, d_q, src_type, B, k_fetch, min_score, d_slots, d_scores, d_counts, d_flags, each);
  if (st != RBK_OK) return st;
  auto copy_back = [&]() -> cudaError_t {
    if (packed) return cudaMemcpyAsync(ix->h_block.p, ix->o_block.p, L.bytes, cudaMemcpyDeviceToHost, ix->stream);
    return cudaMemcpyAsync(ix->h_flags.p, d_flags, sizeof(int) * B, cudaMemcpyDeviceToHost, ix->stream);
  };
  std::vector<int> fails;
  for (;;) {
    CK(copy_back());
    st = ts.round_trip();   // the ONE host round trip of an exact batch
    if (st != RBK_OK) return st;
    if (q.rows && (st = check_gathered(ix)) != RBK_OK) return st;
    fails.clear();
    for (int b = 0; b < B; ++b)
      if (h_flags[b]) fails.push_back(b);
    if (fails.empty() || ix->stats.last_kprime >= kMaxKPrime) break;
    // A proof fails when more rows tie with the k_fetch-th hit (within the scan's error bound) than the
    // candidate margin holds - duplicated chunks, typically.  Before paying an exhaustive fp64 pass per failing
    // query, scan the batch once more at scan speed with the widest margin (k' = 128): groups of up to ~100
    // near-ties then fit among the candidates and the proof goes through.  Results of the queries that had
    // already passed are recomputed to the same values (both passes are exact).
    ix->kprime_override = kMaxKPrime;
    st = run_scan(ix, d_q, src_type, B, k_fetch, min_score, d_slots, d_scores, d_counts, d_flags, nullptr, each);
    ix->kprime_override = 0;
    if (st != RBK_OK) return st;
    ix->stats.retry_batches++;
  }
  if (!fails.empty()) {
    st = run_fallback(ix, fails, k_fetch, min_score, d_slots, d_scores, d_counts, each);
    if (st != RBK_OK) return st;
    // the exhaustive answers are exact by construction: clear the flags the caller may forward
    CK(cudaMemsetAsync(d_flags, 0, sizeof(int) * B, ix->stream));
    if (packed) CK(copy_back());
    st = ts.round_trip();
    if (st != RBK_OK) return st;
  }
  ts.finish(ms_out);
  if (out_slots) L.unpack(ix->h_block.p, out_slots, out_scores, out_counts);
  return RBK_OK;
}

// search_locked of host (q_host) or device (q_dev) queries, exactly one non-null: checks the arguments, takes the lock.
rbk_status search_core(rbk_index* ix, const void* q_host, const void* q_dev, int elem, int B, int query_dim,
                       int k_fetch, double min_score, long long* d_slots, double* d_scores, int* d_counts,
                       int64_t* out_slots, double* out_scores, int32_t* out_counts, float* ms_out,
                       const int32_t* k_each = nullptr, const double* min_each = nullptr) {
  rbk_status st = check_search_args(ix, B, q_host || q_dev, query_dim, k_fetch, min_score);
  if (st != RBK_OK) return st;
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  QuerySource q;
  q.host = q_host;
  q.dev = q_dev;
  return search_locked(ix, q, elem, B, k_fetch, min_score, d_slots, d_scores, d_counts, out_slots, out_scores,
                       out_counts, ms_out, k_each, min_each);
}

}  // namespace

namespace rbk {
namespace impl {
rbk_status search_device_exact(rbk_index* ix, const void* d_q, int elem, int B, int k_fetch, double min_score,
                               long long* d_slots, double* d_scores, int* d_counts, const int32_t* k_each,
                               const double* min_each) {
  return search_core(ix, nullptr, d_q, elem, B, ix ? ix->dim : 0, k_fetch, min_score, d_slots, d_scores, d_counts,
                     nullptr, nullptr, nullptr, nullptr, k_each, min_each);
}

rbk_status check_pairs_args(int64_t slot_base, int64_t size, double min_score, int64_t first_slot, int64_t max_pairs,
                            const void* out_a, const void* out_b, const void* out_scores, const void* n_out,
                            const void* next_slot) {
  if (!out_a || !out_b || !out_scores || !n_out || !next_slot) return fail(RBK_EINVAL, "null output");
  if (min_score != min_score) return fail(RBK_EINVAL, "min_score is NaN");
  if (first_slot < slot_base || first_slot > slot_base + size)
    return fail(RBK_EINVAL, "first_slot must be in [" + std::to_string(slot_base) + ", " +
                                std::to_string(slot_base + size) + "]");
  if (max_pairs < std::max<int64_t>(size, 1))
    return fail(RBK_EINVAL, "max_pairs must be >= max(size(), 1) = " + std::to_string(std::max<int64_t>(size, 1)));
  return RBK_OK;
}

rbk_status similar_pairs_run(const std::vector<rbk_index*>& parts, int64_t end, double min_score, int64_t first_slot,
                             int64_t max_pairs, const std::function<rbk_status(int64_t, int)>& load, int64_t* out_a,
                             int64_t* out_b, double* out_scores, int64_t* n_out, int64_t* next_slot, float* ms_out) {
  const int G = static_cast<int>(parts.size());
  rbk_status st;
  *n_out = 0;
  *next_slot = first_slot;
  if (ms_out) *ms_out = 0.f;
  for (rbk_index* ix : parts) ix->stats.searches++;
  if (first_slot >= end) return RBK_OK;
  std::vector<TimedSearch> ts;
  for (rbk_index* ix : parts) {
    DeviceGuard dg(ix->device);
    ts.push_back(TimedSearch{ix});
    if ((st = ts.back().begin()) != RBK_OK) return st;
  }
  auto each = [&](const std::function<rbk_status(int, rbk_index*)>& f) -> rbk_status {
    for (int d = 0; d < G; ++d) {
      DeviceGuard dg(parts[d]->device);
      rbk_status s2 = f(d, parts[d]);
      if (s2 != RBK_OK) return s2;
    }
    return RBK_OK;
  };
  auto wait_all = [&]() { return each([&](int d, rbk_index*) { return ts[d].round_trip(); }); };
  int64_t n = 0, a0 = first_slot;
  bool full = false;
  std::vector<int64_t> cost;
  while (a0 < end && !full) {
    const int Q = static_cast<int>(std::min<int64_t>(kSlotChunk, end - a0));
    if ((st = each([&](int, rbk_index* ix) { return ensure_query_scratch(ix, Q, 8); })) != RBK_OK) return st;
    if ((st = load(a0, Q)) != RBK_OK) return st;
    if ((st = each([&](int, rbk_index* ix) { return pairs_count(ix, Q, a0, min_score); })) != RBK_OK) return st;
    if ((st = wait_all()) != RBK_OK) return st;   // C_q sizes the candidate buffers and the query groups
    // a query's cost: its candidates, their sort buffer and their packed pairs on every member
    cost.assign(Q, 0);
    for (int q = 0; q < Q; ++q)
      for (rbk_index* ix : parts) cost[q] += ix->h_lcap.p[q] * (large_cand_bytes(true) + 16) + 16;
    const std::vector<std::pair<int, int>> groups = split_by_budget(cost);
    if ((st = each([&](int, rbk_index* ix) { return large_prepare(ix, Q, true, groups); })) != RBK_OK) return st;
    for (const auto& gr : groups) {
      st = each([&](int, rbk_index* ix) { return pairs_emit(ix, gr.first, gr.second, a0, min_score); });
      if (st != RBK_OK || (st = wait_all()) != RBK_OK) return st;
      for (rbk_index* ix : parts)
        if ((st = large_check(ix)) != RBK_OK) return st;
      // the whole query rows that still fit, and each member's share of their pairs (a prefix of its packed pairs)
      int q1 = gr.first;
      int64_t m = 0;
      for (; q1 < gr.second; ++q1) {
        int64_t c = 0;
        for (rbk_index* ix : parts) c += ix->h_pcnt.p[q1 - gr.first];
        if (n + m + c > max_pairs) break;
        m += c;
      }
      std::vector<int64_t> share(G, 0);
      for (int d = 0; d < G; ++d)
        for (int q = gr.first; q < q1; ++q) share[d] += parts[d]->h_pcnt.p[q - gr.first];
      if (m > 0) {
        if ((st = each([&](int d, rbk_index* ix) { return pairs_fetch(ix, share[d]); })) != RBK_OK) return st;
        if ((st = wait_all()) != RBK_OK) return st;
      }
      // every member's list of a query is sorted by (score desc, slot asc), and the members' slots are disjoint
      std::vector<int64_t> at(G, 0);
      for (int q = gr.first; q < q1; ++q) {
        const int64_t o0 = n;
        for (int d = 0; d < G; ++d) {
          const int c = parts[d]->h_pcnt.p[q - gr.first];
          const unsigned char* h = parts[d]->h_block.p;
          memcpy(out_b + n, h + at[d] * 8, sizeof(int64_t) * c);
          memcpy(out_scores + n, h + (share[d] + at[d]) * 8, sizeof(double) * c);
          at[d] += c;
          n += c;
          if (d > 0 && c > 0) {
            std::vector<std::pair<double, int64_t>> v;
            for (int64_t i = o0; i < n; ++i) v.emplace_back(out_scores[i], out_b[i]);
            std::inplace_merge(v.begin(), v.end() - c, v.end(), [](const auto& x, const auto& y) {
              return x.first > y.first || (x.first == y.first && x.second < y.second);
            });
            for (int64_t i = o0; i < n; ++i) {
              out_scores[i] = v[i - o0].first;
              out_b[i] = v[i - o0].second;
            }
          }
        }
        std::fill(out_a + o0, out_a + n, a0 + q);
      }
      if (q1 < gr.second) {   // the buffer is full: the rest of the chunk is answered by the next call
        full = true;
        a0 += q1;
        break;
      }
    }
    if (!full) a0 += Q;
  }
  *n_out = n;
  *next_slot = a0;
  for (int d = 0; d < G; ++d) {
    DeviceGuard dg(parts[d]->device);
    parts[d]->stats.queries += a0 - first_slot;
    float ms = 0.f;
    ts[d].finish(&ms);
    if (ms_out) *ms_out = std::max(*ms_out, ms);
  }
  return RBK_OK;
}

int64_t compact_row_bytes(const rbk_index* ix) {
  return static_cast<int64_t>(ix->dpad) * 2 + static_cast<int64_t>(ix->x_row_bytes()) + 12;
}

rbk_status compact_alloc(rbk_index* ix, int64_t C, int64_t chunk_rows, CompactStage* st) {
  const int64_t n = ix->n_rows, row_bytes = compact_row_bytes(ix);
  const int64_t n_words = (n + 31) / 32, n_blocks = (n_words + 1023) / 1024, n_chunks = (n + chunk_rows - 1) / chunk_rows;
  CK(ix->stage.ensure(static_cast<size_t>(C * row_bytes)));
  CK(ix->cp_map.ensure(static_cast<size_t>(n)));
  CK(ix->cp_scan.ensure(static_cast<size_t>(n_words + n_blocks + n_chunks + 1)));
  unsigned char* p = ix->stage.p;
  st->rows = reinterpret_cast<uint16_t*>(p);
  st->x = p + C * ix->dpad * 2;
  st->norm2 = reinterpret_cast<double*>(p + C * (row_bytes - 12));
  st->inv = reinterpret_cast<float*>(p + C * (row_bytes - 4));
  return RBK_OK;
}

rbk_status compact_map(rbk_index* ix, int64_t chunk_rows, int* h_chunk_pref, int64_t* h_map) {
  const int64_t n = ix->n_rows;
  const int64_t n_words = (n + 31) / 32, n_blocks = (n_words + 1023) / 1024, n_chunks = (n + chunk_rows - 1) / chunk_rows;
  int* word_pref = ix->cp_scan.p;
  int* block_sum = word_pref + n_words;
  int* chunk_pref_d = block_sum + n_blocks;
  CK(launch_compact_map(ix->dead_bits, n, chunk_rows, word_pref, block_sum, ix->cp_map.p, chunk_pref_d, ix->stream));
  ix->stats.kernel_launches += 3;
  CK(cudaMemcpyAsync(h_chunk_pref, chunk_pref_d, sizeof(int) * (n_chunks + 1), cudaMemcpyDeviceToHost, ix->stream));
  if (h_map) CK(cudaMemcpyAsync(h_map, ix->cp_map.p, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, ix->stream));
  return RBK_OK;
}

rbk_status compact_gather(rbk_index* ix, const CompactStage& st, int64_t s0, int64_t n, int64_t rank0) {
  CK(launch_compact_gather(ix->rows, ix->rows_x, ix->x_elem, ix->norm2, ix->inv_norm, ix->cp_map.p, s0, n, rank0,
                           ix->dim, ix->dpad, st.rows, st.x, st.norm2, st.inv, ix->sm_count, ix->stream));
  ix->stats.kernel_launches++;
  return RBK_OK;
}

rbk_status compact_tail(rbk_index* ix, int64_t n_new) {
  // the tail looks like never-appended rows: zero bf16 rows (read by the scan's last tile), NaN 1/||c||, no tombstones
  const int64_t n = ix->n_rows;
  CK(cudaMemsetAsync(ix->rows + n_new * ix->dpad, 0, static_cast<size_t>(n - n_new) * ix->dpad * 2, ix->stream));
  CK(cudaMemsetAsync(ix->inv_norm + n_new, 0xFF, static_cast<size_t>(n - n_new) * 4, ix->stream));
  CK(cudaMemsetAsync(ix->dead_bits, 0, static_cast<size_t>((n + 31) / 32) * 4, ix->stream));
  return RBK_OK;
}

void compact_commit(rbk_index* ix, int64_t n_new) {
  ix->n_rows = n_new;
  ix->n_live = n_new;
  // caches keyed on the corpus: the captured search graph (GraphKey.n_rows) and the corpus tensor map (map_rows) are
  // dropped here so that the next search rebuilds them; the large-k scratch is sized per call from C_q, not from the
  // corpus, and the fallback / exact-scores / debug buffers from n_rows at each call.
  drop_graph(ix);
  ix->tmap_c_rows = -1;
}

uint32_t index_flags(const rbk_index* ix) {
  return (ix->x_elem == 8 ? RBK_INDEX_KEEP_F64 : 0u) | (ix->x_elem == 4 ? RBK_INDEX_KEEP_F32 : 0u) |
         (ix->x_elem == 2 ? RBK_INDEX_KEEP_F32_SPLIT : 0u) |
         (ix->rows_on_host ? RBK_INDEX_ROWS_ON_HOST : 0u) | (ix->scan_f16 ? RBK_INDEX_SCAN_F16 : 0u);
}

rbk_status check_flags(uint32_t flags) {
  constexpr uint32_t kKeep = RBK_INDEX_KEEP_F64 | RBK_INDEX_KEEP_F32 | RBK_INDEX_KEEP_F32_SPLIT;
  if (flags & ~static_cast<uint32_t>(kKeep | RBK_INDEX_ROWS_ON_HOST | RBK_INDEX_SCAN_F16))
    return fail(RBK_EINVAL, "unknown flag");
  if ((flags & (RBK_INDEX_KEEP_F64 | RBK_INDEX_KEEP_F32)) == (RBK_INDEX_KEEP_F64 | RBK_INDEX_KEEP_F32))
    return fail(RBK_EINVAL, "RBK_INDEX_KEEP_F64 and RBK_INDEX_KEEP_F32 exclude each other");
  if ((flags & RBK_INDEX_KEEP_F32_SPLIT) && (flags & (RBK_INDEX_KEEP_F64 | RBK_INDEX_KEEP_F32)))
    return fail(RBK_EINVAL, "RBK_INDEX_KEEP_F32_SPLIT excludes RBK_INDEX_KEEP_F64 and RBK_INDEX_KEEP_F32");
  if ((flags & RBK_INDEX_KEEP_F32_SPLIT) && (flags & RBK_INDEX_SCAN_F16))
    return fail(RBK_EINVAL, "RBK_INDEX_KEEP_F32_SPLIT excludes RBK_INDEX_SCAN_F16: its scan copy holds the high halves");
  // (either keep bit satisfies these two; the messages name the float64 one, as they always have)
  if ((flags & RBK_INDEX_ROWS_ON_HOST) && !(flags & kKeep))
    return fail(RBK_EINVAL, "RBK_INDEX_F64_ON_HOST requires RBK_INDEX_KEEP_F64");
  if ((flags & RBK_INDEX_SCAN_F16) && !(flags & kKeep))
    return fail(RBK_EINVAL, "RBK_INDEX_SCAN_F16 requires RBK_INDEX_KEEP_F64");
  return RBK_OK;
}

rbk_status tier_check(const rbk_index* ix, uint32_t flags) {
  rbk_status st = check_flags(flags);
  if (st != RBK_OK) return st;
  if (((flags & (RBK_INDEX_KEEP_F64 | RBK_INDEX_KEEP_F32 | RBK_INDEX_KEEP_F32_SPLIT)) != 0) != ix->keep_rows())
    return fail(RBK_EINVAL, ix->keep_rows()
                                ? "a tier change keeps the exact rows: RBK_INDEX_KEEP_F64 or RBK_INDEX_KEEP_F32 must stay"
                                : "a tier change cannot add RBK_INDEX_KEEP_F64 or RBK_INDEX_KEEP_F32: this index holds no "
                                  "exact rows");
  return RBK_OK;
}

rbk_status check_f32_exact(rbk_index* ix, const double* src, bool is_device, int64_t n) {
  if (n <= 0) return RBK_OK;
  CK(cudaMemsetAsync(ix->d_counter, 0, sizeof(int), ix->stream));
  if (is_device) {
    CK(launch_find_not_f32(src, n, ix->d_counter, ix->stream));
    ix->stats.kernel_launches++;
  } else {
    const int64_t chunk = std::min<int64_t>(n, (64ll << 20) / 8);
    CK(ix->stage.ensure(static_cast<size_t>(chunk) * 8));
    for (int64_t i0 = 0; i0 < n; i0 += chunk) {
      const int64_t nc = std::min<int64_t>(chunk, n - i0);
      CK(cudaMemcpyAsync(ix->stage.p, src + i0, static_cast<size_t>(nc) * 8, cudaMemcpyHostToDevice, ix->stream));
      CK(launch_find_not_f32(reinterpret_cast<const double*>(ix->stage.p), nc, ix->d_counter, ix->stream));
      ix->stats.kernel_launches++;
    }
  }
  int bad = 0;
  CK(cudaMemcpyAsync(&bad, ix->d_counter, sizeof(int), cudaMemcpyDeviceToHost, ix->stream));
  CK(cudaStreamSynchronize(ix->stream));
  if (bad == 0) return RBK_OK;
  return fail(RBK_ENOTF32, "a value is not exactly a float32, which an RBK_INDEX_KEEP_F32 or KEEP_F32_SPLIT index "
                           "stores (nothing was written)");
}

rbk_status tier_prepare(rbk_index* ix, uint32_t flags, TierPlan* p) {
  *p = TierPlan();
  p->flags = flags;
  p->to_host = (flags & RBK_INDEX_ROWS_ON_HOST) != 0;
  p->x_elem = (flags & RBK_INDEX_KEEP_F32) ? 4 : ((flags & RBK_INDEX_KEEP_F32_SPLIT) ? 2 : 8);
  p->move = p->to_host != ix->rows_on_host || p->x_elem != ix->x_elem;
  p->rescan = ((flags & RBK_INDEX_SCAN_F16) != 0) != ix->scan_f16;
  p->vm_rows = tier_vm_rows(ix, !p->to_host, p->x_elem);
  // searches enqueued earlier finish on the old tier; the corpus-side bound is read once they have
  CK(cudaMemcpyAsync(&p->eps_bits, ix->d_counter + 1, sizeof(int), cudaMemcpyDeviceToHost, ix->stream));
  CK(cudaStreamSynchronize(ix->stream));
  if (ix->cap > p->vm_rows)   // the ceiling falls: exact rows moving to the device, or widened there
    return fail(RBK_ENOMEM, "a capacity of " + std::to_string(ix->cap) + " rows exceeds the " +
                                std::to_string(p->vm_rows) + " this device can hold with these exact rows on it");
  // narrowing: every stored slot, live or tombstoned, must hold float32-exact values (read where the rows are)
  if (ix->x_elem == 8 && p->x_elem != 8) {
    rbk_status st = check_f32_exact(ix, static_cast<const double*>(ix->rows_x), true, ix->n_rows * ix->dim);
    if (st != RBK_OK) return st;
  }
  if (p->move && p->to_host) {
    rbk_status st = alloc_host_rows(static_cast<size_t>(ix->cap) * ix->dim * p->x_elem, &p->host_rows);
    if (st != RBK_OK) return st;
  } else if (p->move) {
    size_t want[rbk_index::kVmBuffers];
    storage_at(ix, p->vm_rows, want, 1, p->x_elem);
    rbk_status st = vm_reserve_range(ix, want[4], &p->vm[4]);
    if (st != RBK_OK) return st;
    storage_at(ix, ix->cap, want, 1, p->x_elem);
    if ((st = vm_map_to(ix, &p->vm[4], want[4])) != RBK_OK) {
      tier_abort(ix, p);
      return st;
    }
  }
  // A ceiling that rises gives buffers 0-3 ranges sized for it, their chunks mapped there too.  Nothing is copied, and
  // no physical memory is added.
  size_t want[rbk_index::kVmBuffers];
  storage_at(ix, p->vm_rows, want, 0);
  for (int i = 0; i < 4; ++i) {
    if (ix->vm[i].reserved >= static_cast<size_t>(round_up(static_cast<int64_t>(want[i]),
                                                            static_cast<int64_t>(ix->vm_gran))))
      continue;   // an index created on a tier with this ceiling or a higher one, or moved there before
    rbk_status st = vm_alias(ix, ix->vm[i], want[i], &p->vm[i]);
    if (st != RBK_OK) {
      tier_abort(ix, p);
      return st;
    }
    p->alias[i] = true;
  }
  return RBK_OK;
}

void tier_abort(rbk_index* ix, TierPlan* p) {
  (void)ix;
  if (p->host_rows) cudaFreeHost(p->host_rows);
  p->host_rows = nullptr;
  for (int i = 0; i < 4; ++i)
    if (p->alias[i]) {
      vm_drop_mapping(&p->vm[i]);   // the chunks stay the index's
      p->alias[i] = false;
    }
  if (p->vm[4].reserved) {
    vm_unmap_from(&p->vm[4], 0);
    vmm_api().MemAddressFree(p->vm[4].base, p->vm[4].reserved);
    p->vm[4] = VmRange();
  }
}

namespace {
// Re-derives the scan copy of rows [0, n_rows) - tombstoned ones too - from the exact rows with the ingest kernels,
// and eps_c_max as the largest angle over them.  1/||c|| stays NaN for tombstoned rows.  A bound that proves nothing (an
// off-band or non-finite row has been stored) stays so until rbk_index_clear, whatever rows the index holds now.
rbk_status tier_rescan(rbk_index* ix, bool f16, int eps_bits) {
  float eps;
  memcpy(&eps, &eps_bits, sizeof eps);
  const int eps0 = eps >= kEpsNone ? eps_bits : 0;
  CK(cudaMemcpyAsync(ix->d_counter + 1, &eps0, sizeof(int), cudaMemcpyHostToDevice, ix->stream));   // pageable: staged
  if (ix->x_elem != 2)   // a split index's scan copy was written with its low halves (tier_commit)
    CK(launch_convert_rows(ix->rows_x, ix->x_elem == 4 ? 1 : 0, ix->n_rows, ix->dim, ix->dpad, ix->rows, nullptr,
                           ix->x_elem, ix->stream, nullptr, nullptr, nullptr, f16));
  CK(launch_row_norms(ix->rows, ix->rows_x, ix->x_elem, 0, ix->n_rows, ix->dim, ix->dpad, ix->inv_norm, ix->norm2,
                      ix->d_counter + 1, ix->stream, nullptr, ix->dead_bits, f16));
  ix->scan_f16 = f16;
  return RBK_OK;
}
}  // namespace

rbk_status tier_commit(rbk_index* ix, TierPlan* p) {
  const bool f16 = (p->flags & RBK_INDEX_SCAN_F16) != 0;
  rbk_status st = RBK_OK;
  // Into or out of the split, the scan copy changes with the exact rows (it holds their high halves): it is rewritten
  // from the new rows, and the norms and the bound with it, once they are in place.
  const bool resplit = p->move && (p->x_elem == 2) != (ix->x_elem == 2);
  if (resplit) p->rescan = true;
  if (p->rescan && !ix->rows_on_host && !resplit) {   // while the exact rows are on the device: no PCIe reads
    if ((st = tier_rescan(ix, f16, p->eps_bits)) != RBK_OK) return st;
    p->rescan = false;
  }
  if (p->move) {
    void* dst = p->to_host ? p->host_rows : reinterpret_cast<void*>(p->vm[4].base);
    const int64_t n_el = ix->n_rows * ix->dim;
    if (n_el > 0 && p->x_elem == ix->x_elem)   // a move between the device and the host: UVA picks the direction
      CK(cudaMemcpyAsync(dst, ix->rows_x, static_cast<size_t>(n_el) * ix->x_elem, cudaMemcpyDefault, ix->stream));
    else if (n_el > 0 && p->x_elem == 2)       // into the split: both halves from the float32-exact rows
      CK(launch_convert_rows(ix->rows_x, ix->x_elem == 4 ? 1 : 0, ix->n_rows, ix->dim, ix->dpad, ix->rows, dst, 2,
                             ix->stream));
    else if (n_el > 0)                         // widen or narrow on the device, reading and writing where the rows are
      CK(launch_convert_exact(ix->rows_x, ix->x_elem, dst, p->x_elem, n_el, ix->stream, ix->rows, ix->dim, ix->dpad));
    CK(cudaStreamSynchronize(ix->stream));
    if (ix->rows_on_host) {
      cudaFreeHost(ix->rows_x);
    } else {
      vm_unmap_from(&ix->vm[4], 0);
      if (ix->vm[4].reserved) vmm_api().MemAddressFree(ix->vm[4].base, ix->vm[4].reserved);
      ix->vm[4] = VmRange();
    }
    if (p->to_host) {
      ix->rows_x = p->host_rows;
      p->host_rows = nullptr;
    } else {
      ix->vm[4] = std::move(p->vm[4]);
      p->vm[4] = VmRange();
      ix->rows_x = reinterpret_cast<void*>(ix->vm[4].base);
    }
    ix->rows_on_host = p->to_host;
    ix->x_elem = p->x_elem;
  }
  for (int i = 0; i < 4; ++i) {
    if (!p->alias[i]) continue;
    vm_drop_mapping(&ix->vm[i]);   // the old addresses; the chunks now belong to the new range
    ix->vm[i] = std::move(p->vm[i]);
    p->vm[i] = VmRange();
    p->alias[i] = false;
  }
  ix->rows = reinterpret_cast<uint16_t*>(ix->vm[0].base);
  ix->inv_norm = reinterpret_cast<float*>(ix->vm[1].base);
  ix->norm2 = reinterpret_cast<double*>(ix->vm[2].base);
  ix->dead_bits = reinterpret_cast<unsigned int*>(ix->vm[3].base);
  ix->vm_rows = p->vm_rows;
  if (p->rescan && (st = tier_rescan(ix, f16, p->eps_bits)) != RBK_OK) return st;
  CK(cudaStreamSynchronize(ix->stream));
  // every cache keyed on the old tier or the old pointers: the captured graph (its scan instantiation and pointers)
  // and the corpus tensor map (its data type and base); the other scratch buffers hold no corpus pointer
  drop_graph(ix);
  ix->tmap_c_rows = -1;
  return RBK_OK;
}
}  // namespace impl
}  // namespace rbk

// =========================================================================== C ABI
extern "C" {

int rbk_abi_version(void) { return RBK_ABI_VERSION; }
const char* rbk_last_error(void) { return rbk::impl::last_error(); }

rbk_status rbk_index_create(int32_t dim, int32_t device, int64_t capacity_hint, rbk_index** out) {
  return rbk_index_create_ex(dim, device, capacity_hint, 0, out);
}

rbk_status rbk_index_create_ex(int32_t dim, int32_t device, int64_t capacity_hint, uint32_t flags, rbk_index** out) {
  if (!out) return fail(RBK_EINVAL, "out is null");
  *out = nullptr;
  rbk_status fst = check_flags(flags);
  if (fst != RBK_OK) return fst;
  if (dim < 1 || dim > RBK_MAX_DIM) return fail(RBK_EINVAL, "dim out of range");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(RBK_ECUDA, std::string("no CUDA device (this engine has no CPU path): ") +
                               (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
  if (device < 0 || device >= ndev) return fail(RBK_EINVAL, "device ordinal out of range");
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(RBK_ECUDA, std::string("this build targets sm_90a (Hopper H100); device is ") + prop.name);
  DeviceGuard dg(device);
  rbk_index* ix = new (std::nothrow) rbk_index();
  if (!ix) return fail(RBK_ENOMEM, "out of host memory");
  ix->dim = dim;
  // row pitch = whole 128-byte lines (64-element k-blocks): no TMA box hangs over the end of a row
  ix->dpad = static_cast<int>(round_up(dim, kBlockK));
  ix->device = device;
  ix->x_elem = (flags & RBK_INDEX_KEEP_F64)         ? 8
               : (flags & RBK_INDEX_KEEP_F32)       ? 4
               : (flags & RBK_INDEX_KEEP_F32_SPLIT) ? 2
                                                    : 0;
  ix->rows_on_host = (flags & RBK_INDEX_ROWS_ON_HOST) != 0;
  ix->scan_f16 = (flags & RBK_INDEX_SCAN_F16) != 0;
  ix->sm_count = prop.multiProcessorCount;
  memset(&ix->stats, 0, sizeof ix->stats);
  ix->stats.sm_count = ix->sm_count;
  e = cudaStreamCreateWithFlags(&ix->own_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    delete ix;
    return cuda_fail(e, "cudaStreamCreate");
  }
  if ((e = cudaEventCreate(&ix->ev_start)) != cudaSuccess || (e = cudaEventCreate(&ix->ev_stop)) != cudaSuccess) {
    rbk_index_destroy(ix);
    return cuda_fail(e, "cudaEventCreate");
  }
  ix->stream = ix->own_stream;
  e = cudaMalloc(reinterpret_cast<void**>(&ix->d_counter), 2 * sizeof(int));
  if (e == cudaSuccess) e = cudaMemset(ix->d_counter, 0, 2 * sizeof(int));
  if (e != cudaSuccess) {
    rbk_index_destroy(ix);
    return cuda_fail(e, "cudaMalloc");
  }
  rbk_status st = vm_reserve(ix, prop.totalGlobalMem);
  if (st == RBK_OK) st = ensure_capacity(ix, std::max<int64_t>(capacity_hint, 1024));
  if (st != RBK_OK) {
    rbk_index_destroy(ix);
    return st;
  }
  *out = ix;
  return RBK_OK;
}

void rbk_index_destroy(rbk_index* ix) {
  if (!ix) return;
  {
    DeviceGuard dg(ix->device);
    if (ix->stream) cudaStreamSynchronize(ix->stream);
    vm_free(ix);
    if (ix->rows_on_host) cudaFreeHost(ix->rows_x);
    cudaFree(ix->d_counter);
    release_scratch(ix);
    if (ix->ev_start) cudaEventDestroy(ix->ev_start);
    if (ix->ev_stop) cudaEventDestroy(ix->ev_stop);
    for (auto& pr : ix->tev)
      for (cudaEvent_t e : pr)
        if (e) cudaEventDestroy(e);
    if (ix->own_stream) cudaStreamDestroy(ix->own_stream);
  }
  delete ix;
}

rbk_status rbk_index_set_stream(rbk_index* ix, void* cuda_stream) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  CK(cudaStreamSynchronize(ix->stream));
  ix->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ix->own_stream;
  return RBK_OK;
}

rbk_status rbk_index_set_slot_base(rbk_index* ix, int64_t slot_base) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  if (slot_base < 0) return fail(RBK_EINVAL, "slot_base must be >= 0");
  std::lock_guard<std::mutex> lk(ix->mu);
  ix->slot.base = slot_base;
  return RBK_OK;
}

rbk_status rbk_index_append_f64(rbk_index* ix, const double* rows, int64_t n, int64_t* first) {
  return append_rows(ix, rows, false, 8, n, first);
}
rbk_status rbk_index_append_f32(rbk_index* ix, const float* rows, int64_t n, int64_t* first) {
  return append_rows(ix, rows, false, 4, n, first);
}
rbk_status rbk_index_append_bf16(rbk_index* ix, const uint16_t* rows, int64_t n, int64_t* first) {
  return append_rows(ix, rows, false, 2, n, first);
}
rbk_status rbk_index_append_bf16_device(rbk_index* ix, const void* dev_rows, int64_t n, int64_t* first) {
  return append_rows(ix, dev_rows, true, 2, n, first);
}
rbk_status rbk_index_append_f64_device(rbk_index* ix, const void* dev_rows, int64_t n, int64_t* first) {
  return append_rows(ix, dev_rows, true, 8, n, first);
}

rbk_status rbk_index_overwrite_f64_batch(rbk_index* ix, const int64_t* slots, int64_t n, const double* rows) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  if (n < 0 || (n > 0 && (!slots || !rows))) return fail(RBK_EINVAL, "bad argument");
  if (n == 0) return RBK_OK;
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  for (int64_t i = 0; i < n; ++i)
    if (slots[i] < 0 || slots[i] >= ix->n_rows) return fail(RBK_EINVAL, "slot out of range");
  // The same slot twice in one batch is Map.set twice: the LAST value wins (and two thread blocks scattering into one
  // row would race).  Keep each slot's last occurrence; the common case (no repeats) copies nothing.
  std::vector<int64_t> u_slots;
  std::vector<double> u_rows;
  if (n > 1) {
    std::unordered_map<int64_t, int64_t> last;
    last.reserve(static_cast<size_t>(n) * 2);
    for (int64_t i = 0; i < n; ++i) last[slots[i]] = i;
    if (static_cast<int64_t>(last.size()) != n) {
      u_slots.reserve(last.size());
      u_rows.resize(last.size() * static_cast<size_t>(ix->dim));
      for (int64_t i = 0; i < n; ++i) {
        if (last[slots[i]] != i) continue;
        memcpy(u_rows.data() + u_slots.size() * static_cast<size_t>(ix->dim), rows + static_cast<size_t>(i) * ix->dim,
               static_cast<size_t>(ix->dim) * 8);
        u_slots.push_back(slots[i]);
      }
      slots = u_slots.data();
      rows = u_rows.data();
      n = static_cast<int64_t>(u_slots.size());
    }
  }
  // float32 exact rows: every value is checked before the first slot is written
  if (ix->f32_rows()) {
    rbk_status st = check_f32_exact(ix, rows, false, n * ix->dim);
    if (st != RBK_OK) return st;
  }
  // one H2D of the slots, one of the rows (chunked through the staging buffer), two kernels per chunk that scatter
  // into the named slots and skip tombstoned ones on the device, ONE host round trip for the whole batch
  const size_t row_bytes = static_cast<size_t>(ix->dim) * 8;
  const int64_t chunk_rows = std::max<int64_t>(1, std::min<int64_t>(n, (64ll << 20) / static_cast<int64_t>(row_bytes)));
  CK(ix->stage.ensure(static_cast<size_t>(chunk_rows) * row_bytes));
  CK(ix->d_slots.ensure(static_cast<size_t>(n)));
  CK(cudaMemcpyAsync(ix->d_slots.p, slots, sizeof(int64_t) * n, cudaMemcpyHostToDevice, ix->stream));
  CK(cudaMemsetAsync(ix->d_counter, 0, sizeof(int), ix->stream));
  for (int64_t r0 = 0; r0 < n; r0 += chunk_rows) {
    const int64_t nr = std::min<int64_t>(chunk_rows, n - r0);
    CK(cudaMemcpyAsync(ix->stage.p, reinterpret_cast<const unsigned char*>(rows) + static_cast<size_t>(r0) * row_bytes,
                       static_cast<size_t>(nr) * row_bytes, cudaMemcpyHostToDevice, ix->stream));
    CK(launch_convert_rows(ix->stage.p, 0, nr, ix->dim, ix->dpad, ix->rows, ix->rows_x, ix->x_elem, ix->stream,
                           ix->d_slots.p + r0, ix->dead_bits, ix->d_counter, ix->scan_f16));
    CK(launch_row_norms(ix->rows, ix->rows_x, ix->x_elem, 0, nr, ix->dim, ix->dpad, ix->inv_norm, ix->norm2,
                        ix->d_counter + 1, ix->stream, ix->d_slots.p + r0, ix->dead_bits, ix->scan_f16));
    ix->stats.kernel_launches += ix->keep_rows() ? 3 : 2;
  }
  int dead = 0;
  CK(cudaMemcpyAsync(&dead, ix->d_counter, sizeof(int), cudaMemcpyDeviceToHost, ix->stream));
  CK(cudaStreamSynchronize(ix->stream));
  if (dead > 0) {
    // a tombstoned slot stays dead: the host never overwrites a deleted id (S9b: a re-added id is appended)
    char buf[96];
    snprintf(buf, sizeof buf, "slot is tombstoned (%d of %lld rows skipped)", dead, static_cast<long long>(n));
    return fail(RBK_EINVAL, buf);
  }
  return RBK_OK;
}

rbk_status rbk_index_overwrite_f64(rbk_index* ix, int64_t slot, const double* row) {
  if (!row) return fail(RBK_EINVAL, "null argument");
  return rbk_index_overwrite_f64_batch(ix, &slot, 1, row);
}

rbk_status rbk_index_tombstone(rbk_index* ix, const int64_t* slots, int64_t n) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  if (n < 0 || (n > 0 && !slots)) return fail(RBK_EINVAL, "bad slots argument");
  if (n == 0) return RBK_OK;
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  for (int64_t i = 0; i < n; ++i)
    if (slots[i] < 0 || slots[i] >= ix->n_rows) return fail(RBK_EINVAL, "slot out of range");
  CK(ix->d_slots.ensure(static_cast<size_t>(n)));
  CK(cudaMemcpyAsync(ix->d_slots.p, slots, sizeof(int64_t) * n, cudaMemcpyHostToDevice, ix->stream));
  CK(cudaMemsetAsync(ix->d_counter, 0, sizeof(int), ix->stream));
  CK(launch_tombstone(ix->d_slots.p, n, ix->n_rows, ix->inv_norm, ix->dead_bits, ix->d_counter, ix->stream));
  ix->stats.kernel_launches++;
  int killed = 0;
  CK(cudaMemcpyAsync(&killed, ix->d_counter, sizeof(int), cudaMemcpyDeviceToHost, ix->stream));
  CK(cudaStreamSynchronize(ix->stream));
  ix->n_live -= killed;
  return RBK_OK;
}

rbk_status rbk_index_clear(rbk_index* ix) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  CK(cudaMemsetAsync(ix->inv_norm, 0xFF, static_cast<size_t>(inv_norm_len(ix->cap)) * 4, ix->stream));
  CK(cudaMemsetAsync(ix->dead_bits, 0, static_cast<size_t>((ix->cap + 31) / 32) * 4, ix->stream));
  CK(cudaMemsetAsync(ix->d_counter, 0, 2 * sizeof(int), ix->stream));   // also resets the corpus-side error bound
  CK(cudaStreamSynchronize(ix->stream));
  ix->n_rows = 0;
  ix->n_live = 0;
  return RBK_OK;
}

rbk_status rbk_index_compact(rbk_index* ix, int64_t* old_to_new, int64_t old_to_new_len) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  const int64_t n = ix->n_rows, n_live = ix->n_live;
  if (old_to_new && old_to_new_len < n) return fail(RBK_EINVAL, "old_to_new_len is shorter than size()");
  if (ix->slot.block != 0)   // block-cyclic rows: moving them would break the group's slot layout
    return fail(RBK_EINVAL, "compaction is not available for a member of a device group (use rbk_group_compact)");
  if (n_live == n) {         // no tombstones (or an empty index): nothing moves, every cache stays valid
    for (int64_t s = 0; old_to_new && s < n; ++s) old_to_new[s] = s;
    return RBK_OK;
  }
  // Staging chunk: whole 32-row words, 64 MB (the append path's staging size) of packed rows.
  const int64_t C = std::min(round_up(n, 32), std::max<int64_t>(32, (64ll << 20) / compact_row_bytes(ix) / 32 * 32));
  const int64_t n_chunks = (n + C - 1) / C;
  // every allocation before the first row moves: RBK_ENOMEM leaves the index untouched
  CompactStage st;
  rbk_status s = compact_alloc(ix, C, C, &st);
  if (s != RBK_OK) return s;
  std::vector<int> chunk_pref(static_cast<size_t>(n_chunks + 1));
  s = compact_map(ix, C, chunk_pref.data(), old_to_new);
  if (s != RBK_OK) return s;
  CK(cudaStreamSynchronize(ix->stream));
  if (chunk_pref[n_chunks] != n_live)
    return fail(RBK_ECUDA, "compaction: the tombstone bits count " + std::to_string(chunk_pref[n_chunks]) +
                               " live rows, the index " + std::to_string(n_live) + " (the index was not changed)");
  // In place, stable, one chunk of sources at a time.  Chunk [s0, s1) holds L live rows that land at [d0, d0 + L) with
  // d0 + L <= s1: the copies overwrite only rows of this chunk and of earlier ones, all already staged, never a
  // source of a later chunk.  Chunks before the first tombstone (d0 == s0, L == s1 - s0) do not move.
  for (int64_t c = 0; c < n_chunks; ++c) {
    const int64_t s0 = c * C, s1 = std::min(n, s0 + C);
    const int64_t d0 = chunk_pref[c], L = chunk_pref[c + 1] - d0;
    if ((d0 == s0 && L == s1 - s0) || L == 0) continue;
    s = compact_gather(ix, st, s0, s1 - s0, d0);
    if (s != RBK_OK) return s;
    CK(cudaMemcpyAsync(ix->rows + d0 * ix->dpad, st.rows, static_cast<size_t>(L) * ix->dpad * 2,
                       cudaMemcpyDeviceToDevice, ix->stream));
    if (ix->keep_rows())   // device or mapped host rows (RBK_INDEX_ROWS_ON_HOST): UVA picks the direction
      CK(cudaMemcpyAsync(static_cast<unsigned char*>(ix->rows_x) + d0 * ix->x_row_bytes(), st.x,
                         static_cast<size_t>(L) * ix->x_row_bytes(), cudaMemcpyDefault, ix->stream));
    CK(cudaMemcpyAsync(ix->norm2 + d0, st.norm2, static_cast<size_t>(L) * 8, cudaMemcpyDeviceToDevice, ix->stream));
    CK(cudaMemcpyAsync(ix->inv_norm + d0, st.inv, static_cast<size_t>(L) * 4, cudaMemcpyDeviceToDevice, ix->stream));
  }
  s = compact_tail(ix, n_live);
  if (s != RBK_OK) return s;
  CK(cudaStreamSynchronize(ix->stream));
  compact_commit(ix, n_live);
  return RBK_OK;
}

rbk_status rbk_index_trim(rbk_index* ix) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  CK(cudaStreamSynchronize(ix->stream));   // searches enqueued earlier finish before anything they read goes away
  // the capacity of a new index holding size() rows; rows, 1/||c|| (NaN), norm2 and tombstone bits beyond size() are
  // never-appended rows already, so nothing below the new capacity changes
  const int64_t tcap = round_up(std::max<int64_t>(ix->n_rows, 1024), kBlockN);
  if (tcap < ix->cap) {
    if (ix->rows_on_host) {
      rbk_status st = realloc_host_rows(ix, tcap);
      if (st != RBK_OK) return st;
    }
    size_t keep[rbk_index::kVmBuffers];
    storage_at(ix, tcap, keep);
    for (int i = 0; i < rbk_index::kVmBuffers; ++i) vm_unmap_from(&ix->vm[i], keep[i]);
    ix->cap = tcap;
  }
  release_scratch(ix);
  ix->tmap_c_rows = -1;
  return RBK_OK;
}

uint32_t rbk_index_flags(const rbk_index* ix) { return ix ? index_flags(ix) : 0u; }

rbk_status rbk_index_set_tier(rbk_index* ix, uint32_t flags) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  std::lock_guard<std::mutex> lk(ix->mu);
  if (ix->slot.block != 0)
    return fail(RBK_EINVAL, "a tier change is not available for a member of a device group (use rbk_group_set_tier)");
  rbk_status st = tier_check(ix, flags);
  if (st != RBK_OK || flags == index_flags(ix)) return st;
  DeviceGuard dg(ix->device);
  TierPlan plan;
  if ((st = tier_prepare(ix, flags, &plan)) != RBK_OK) return st;
  if ((st = tier_commit(ix, &plan)) != RBK_OK) tier_abort(ix, &plan);   // a CUDA error: release what was not taken over
  return st;
}

int64_t rbk_index_count(const rbk_index* ix) { return ix ? ix->n_live : 0; }
int64_t rbk_index_size(const rbk_index* ix) { return ix ? ix->n_rows : 0; }
int32_t rbk_index_dim(const rbk_index* ix) { return ix ? ix->dim : 0; }

rbk_status rbk_index_storage_bytes(const rbk_index* ix, int64_t* device_bytes, int64_t* pinned_host_bytes) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  // the buffers of ensure_capacity: rows | inv_norm | norm2 | dead_bits | f64 rows
  size_t bytes[rbk_index::kVmBuffers];
  storage_at(ix, ix->cap, bytes);
  int64_t dev = 0;
  for (size_t b : bytes) dev += static_cast<int64_t>(b);
  if (device_bytes) *device_bytes = dev;
  if (pinned_host_bytes) *pinned_host_bytes = ix->rows_on_host ? ix->cap * static_cast<int64_t>(ix->x_row_bytes()) : 0;
  return RBK_OK;
}

namespace {
rbk_status read_rows(rbk_index* ix, int64_t first, int64_t n, uint16_t* out, bool f16) {
  if (!ix || (n > 0 && !out)) return fail(RBK_EINVAL, "null argument");
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  if (ix->scan_f16 != f16)
    return fail(RBK_EINVAL, ix->scan_f16 ? "this index stores fp16 rows (RBK_INDEX_SCAN_F16): use rbk_index_read_rows_f16"
                                         : "this index stores bf16 rows: use rbk_index_read_rows_bf16");
  if (first < 0 || n < 0 || first + n > ix->n_rows) return fail(RBK_EINVAL, "row range out of bounds");
  if (n == 0) return RBK_OK;
  CK(cudaMemcpy2DAsync(out, static_cast<size_t>(ix->dim) * 2, ix->rows + static_cast<size_t>(first) * ix->dpad,
                       static_cast<size_t>(ix->dpad) * 2, static_cast<size_t>(ix->dim) * 2, static_cast<size_t>(n),
                       cudaMemcpyDeviceToHost, ix->stream));
  CK(cudaStreamSynchronize(ix->stream));
  return RBK_OK;
}
}  // namespace

rbk_status rbk_index_read_rows_bf16(rbk_index* ix, int64_t first, int64_t n, uint16_t* out) {
  return read_rows(ix, first, n, out, false);
}
rbk_status rbk_index_read_rows_f16(rbk_index* ix, int64_t first, int64_t n, uint16_t* out) {
  return read_rows(ix, first, n, out, true);
}

rbk_status rbk_index_search_f64(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                                double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                                float* kernel_ms_out) {
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  return search_core(ix, queries, nullptr, 8, B, query_dim, k_fetch, min_score, nullptr, nullptr, nullptr, out_slots,
                     out_scores, out_counts, kernel_ms_out);
}
rbk_status rbk_index_search_f32(rbk_index* ix, const float* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                                double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                                float* kernel_ms_out) {
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  return search_core(ix, queries, nullptr, 4, B, query_dim, k_fetch, min_score, nullptr, nullptr, nullptr, out_slots,
                     out_scores, out_counts, kernel_ms_out);
}
rbk_status rbk_index_search_device(rbk_index* ix, const void* dev_queries_f32, int32_t B, int32_t k_fetch,
                                   double min_score, void* dev_out_slots, void* dev_out_scores,
                                   void* dev_out_counts) {
  if (B > 0 && (!dev_queries_f32 || !dev_out_slots || !dev_out_scores || !dev_out_counts))
    return fail(RBK_EINVAL, "null device pointer");
  return search_core(ix, nullptr, dev_queries_f32, 4, B, ix ? ix->dim : 0, k_fetch, min_score,
                     static_cast<long long*>(dev_out_slots), static_cast<double*>(dev_out_scores),
                     static_cast<int*>(dev_out_counts), nullptr, nullptr, nullptr, nullptr);
}

namespace {
// The large-k search for k_fetch in [1, max_k] (rbk_index_impl.h): the count scan, one wait, then per query group
// the emit scan and the cut into o_block, its D2H into the pinned h_block, a wait, and the copy into the caller's rows
// of k_fetch entries.  k_each / min_each (host [B], nullable; checked by the caller): a search_each call's own cut and
// threshold per query, k_fetch their largest k; each query is then cut at its own k_eff.
// large_locked: the caller holds the lock, has the device current and has checked the arguments; the queries come from
// q (float64 ones).
rbk_status large_locked(rbk_index* ix, const QuerySource& q, int32_t B, int32_t k_fetch, double min_score,
                        int64_t* out_slots, double* out_scores, int32_t* out_counts, float* kernel_ms_out,
                        const int32_t* k_each = nullptr, const double* min_each = nullptr) {
  rbk_status st;
  if (kernel_ms_out) *kernel_ms_out = 0.f;
  if (B == 0) {
    ix->stats.searches++;
    return RBK_OK;
  }
  const bool sorted = k_fetch > RBK_MAX_K_FETCH_LARGE;
  // the sort's buffers are sized by k_eff: no query can have more hits than there are live rows
  const int k_eff = sorted ? static_cast<int>(std::min<int64_t>(k_fetch, ix->n_live)) : k_fetch;
  std::vector<int32_t> k_eff_each;   // search_each: every query's own k_eff, by the same rule
  if (k_each)
    for (int b = 0; b < B; ++b)
      k_eff_each.push_back(sorted ? static_cast<int32_t>(std::min<int64_t>(k_each[b], ix->n_live)) : k_each[b]);
  if (k_eff == 0) {
    fill_result_tail(out_slots, out_scores, B, k_fetch, 0);
    memset(out_counts, 0, sizeof(int32_t) * B);
    ix->stats.searches++;
    ix->stats.queries += B;
    return RBK_OK;
  }
  st = ensure_query_scratch(ix, B, 8);
  if (st != RBK_OK) return st;
  TimedSearch ts{ix};
  st = ts.begin();
  if (st != RBK_OK) return st;
  QueryCuts each;
  if (k_each && (st = upload_cuts(ix, B, k_eff_each.data(), min_each, &each)) != RBK_OK) return st;
  const void* d_q = nullptr;
  if ((st = load_queries(ix, q, B, 8, &d_q)) != RBK_OK) return st;
  st = large_count(ix, d_q, B, k_eff, min_score, each);
  if (st != RBK_OK) return st;
  CK(cudaStreamSynchronize(ix->stream));   // C_q sizes the candidate buffers and the query groups
  if (q.rows && (st = check_gathered(ix)) != RBK_OK) return st;
  std::vector<int64_t> cost(B);
  for (int b = 0; b < B; ++b) cost[b] = ix->h_lcap.p[b] * large_cand_bytes(sorted) + large_result_bytes(k_eff);
  const std::vector<std::pair<int, int>> groups = split_by_budget(cost);
  st = large_prepare(ix, B, sorted, groups);
  if (st != RBK_OK) return st;
  int max_group = 0;
  for (const auto& gr : groups) max_group = std::max(max_group, gr.second - gr.first);
  // no flags: every answer is exact by construction
  const size_t blk = ResultBlock(max_group, k_eff).off_counts + sizeof(int32_t) * max_group;
  CK(ix->o_block.ensure(blk));
  CK(ix->h_block.ensure(blk));
  for (const auto& gr : groups) {
    const ResultBlock R(gr.second - gr.first, k_eff);
    unsigned char* base = ix->o_block.p;
    st = large_emit(ix, gr.first, gr.second, sorted, k_eff, min_score, R.slots(base), R.scores(base), R.counts(base),
                    each);
    if (st == RBK_OK && gr.second == B) st = large_finish(ix);   // the overflow count rides the last round trip
    if (st != RBK_OK) return st;
    CK(cudaMemcpyAsync(ix->h_block.p, base, R.off_counts + sizeof(int32_t) * R.B, cudaMemcpyDeviceToHost, ix->stream));
    st = ts.round_trip();
    if (st != RBK_OK) return st;
    const size_t o = static_cast<size_t>(gr.first) * k_fetch;
    R.unpack_rows(ix->h_block.p, k_fetch, out_slots + o, out_scores + o, out_counts + gr.first);
  }
  st = large_check(ix);
  if (st != RBK_OK) return st;
  ts.finish(kernel_ms_out);
  return RBK_OK;
}

rbk_status search_large(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                        double min_score, int max_k, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                        float* kernel_ms_out, const int32_t* k_each = nullptr, const double* min_each = nullptr) {
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  rbk_status st = check_search_args(ix, B, queries != nullptr, query_dim, k_fetch, min_score, max_k);
  if (st != RBK_OK) return st;
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  QuerySource q;
  q.host = queries;
  return large_locked(ix, q, B, k_fetch, min_score, out_slots, out_scores, out_counts, kernel_ms_out, k_each,
                      min_each);
}
}  // namespace

rbk_status rbk_index_search_large_f64(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim,
                                      int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                      int32_t* out_counts, float* kernel_ms_out) {
  return search_large(ix, queries, B, query_dim, k_fetch, min_score, RBK_MAX_K_FETCH_LARGE, out_slots, out_scores,
                      out_counts, kernel_ms_out);
}

rbk_status rbk_index_search_unbounded_f64(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim,
                                          int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                          int32_t* out_counts, float* kernel_ms_out) {
  return search_large(ix, queries, B, query_dim, k_fetch, min_score, INT32_MAX, out_slots, out_scores, out_counts,
                      kernel_ms_out);
}

rbk_status rbk_index_search_each_f64(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim,
                                     const int32_t* k_fetch, const double* min_score, int64_t* out_slots,
                                     double* out_scores, int32_t* out_counts, float* kernel_ms_out) {
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  int K = 0;
  rbk_status st = check_each_args(ix, B, queries != nullptr, query_dim, k_fetch, min_score, &K);
  if (st != RBK_OK) return st;
  if (B == 0) {
    if (kernel_ms_out) *kernel_ms_out = 0.f;
    std::lock_guard<std::mutex> lk(ix->mu);
    ix->stats.searches++;
    return RBK_OK;
  }
  // One route for the whole batch, picked by its largest k: the scan's top-k' with every query cut at its own k, or
  // the two-scan large-k pipeline for every query (exact on either route, so a small k loses nothing there).  The
  // scalar min_score of both is unused: every kernel that applies one reads the query's own.
  if (K <= RBK_MAX_K_FETCH)
    return search_core(ix, queries, nullptr, 8, B, query_dim, K, -INFINITY, nullptr, nullptr, nullptr, out_slots,
                       out_scores, out_counts, kernel_ms_out, k_fetch, min_score);
  return search_large(ix, queries, B, query_dim, K, -INFINITY, INT32_MAX, out_slots, out_scores, out_counts,
                      kernel_ms_out, k_fetch, min_score);
}

rbk_status rbk_index_search_slots_f64(rbk_index* ix, const int64_t* query_slots, int32_t B, const int32_t* k_fetch,
                                      const double* min_score, int64_t* out_slots, double* out_scores,
                                      int32_t* out_counts, float* kernel_ms_out) {
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  int K = 0;
  rbk_status st = check_each_args(ix, B, query_slots != nullptr, ix ? ix->dim : 0, k_fetch, min_score, &K);
  if (st != RBK_OK) return st;
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  if (kernel_ms_out) *kernel_ms_out = 0.f;
  std::vector<int64_t> rows(B);
  for (int b = 0; b < B; ++b) {
    rows[b] = ix->slot.local(query_slots[b]);
    if (rows[b] < 0 || rows[b] >= ix->n_rows)
      return fail(RBK_EINVAL, "query_slots[" + std::to_string(b) + "] is not a slot of this index");
  }
  // every slot is held, so none is live: the large-k route would answer before its gather could say so
  if (B > 0 && ix->n_live == 0) return fail(RBK_EINVAL, "query slot is tombstoned (the index has no live row)");
  // one call is one search, however many chunks it takes
  const int64_t searches = ix->stats.searches + 1;
  std::vector<int64_t> c_slots;
  std::vector<double> c_scores;
  for (int c0 = 0; c0 < B; c0 += kSlotChunk) {
    const int Bc = std::min(kSlotChunk, B - c0);
    const int Kc = *std::max_element(k_fetch + c0, k_fetch + c0 + Bc);
    const size_t o = static_cast<size_t>(c0) * K;
    // a chunk's rows are Kc entries long: straight into the caller's rows when that is K, else through c_*
    if (Kc < K) {
      c_slots.resize(static_cast<size_t>(Bc) * Kc);
      c_scores.resize(static_cast<size_t>(Bc) * Kc);
    }
    int64_t* cs = Kc < K ? c_slots.data() : out_slots + o;
    double* cd = Kc < K ? c_scores.data() : out_scores + o;
    QuerySource q;
    q.rows = rows.data() + c0;
    float ms = 0.f;
    // the route rbk_index_search_each_f64 takes for the chunk's largest k
    st = Kc <= RBK_MAX_K_FETCH
             ? search_locked(ix, q, 8, Bc, Kc, -INFINITY, nullptr, nullptr, nullptr, cs, cd, out_counts + c0, &ms,
                             k_fetch + c0, min_score + c0)
             : large_locked(ix, q, Bc, Kc, -INFINITY, cs, cd, out_counts + c0, &ms, k_fetch + c0, min_score + c0);
    if (st != RBK_OK) return st;
    if (Kc < K) {
      for (int b = 0; b < Bc; ++b) {
        memcpy(out_slots + o + static_cast<size_t>(b) * K, cs + static_cast<size_t>(b) * Kc, sizeof(int64_t) * Kc);
        memcpy(out_scores + o + static_cast<size_t>(b) * K, cd + static_cast<size_t>(b) * Kc, sizeof(double) * Kc);
      }
      fill_result_tail(out_slots + o, out_scores + o, Bc, K, Kc);
    }
    if (kernel_ms_out) *kernel_ms_out += ms;
  }
  ix->stats.searches = searches;
  return RBK_OK;
}

rbk_status rbk_index_search_mmr_f64(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim,
                                    const int32_t* k, const int32_t* fetch_k, const double* lambda_mult,
                                    const double* min_score, int64_t* out_slots, double* out_scores,
                                    int32_t* out_counts, float* kernel_ms_out) {
  int K = 0;
  rbk_status st = check_mmr_args(ix, B, queries != nullptr, query_dim, k, fetch_k, lambda_mult, min_score, out_slots,
                                 out_scores, out_counts, &K);
  if (st != RBK_OK) return st;
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  if (kernel_ms_out) *kernel_ms_out = 0.f;
  // one call is one search, however many chunks it takes
  const int64_t searches = ix->stats.searches + 1;
  // the candidates' rows, gathered where the index keeps them (a candidate is live, so the gather must count no dead row)
  std::vector<int64_t> rows;
  MmrStage stage;
  stage.host = [&](const int64_t* slots, int n) -> rbk_status {
    rows.resize(n);
    for (int i = 0; i < n; ++i) rows[i] = ix->slot.local(slots[i]);
    return RBK_OK;
  };
  stage.device = [&](int n) -> rbk_status { return gather_queries(ix, rows.data(), n); };
  std::vector<int64_t> c_slots;
  std::vector<double> c_scores;
  std::vector<int32_t> c_counts;
  for (int c0 = 0; c0 < B; c0 += kSlotChunk) {
    const int Bc = std::min(kSlotChunk, B - c0);
    const int F = *std::max_element(fetch_k + c0, fetch_k + c0 + Bc);
    c_slots.resize(static_cast<size_t>(Bc) * F);
    c_scores.resize(static_cast<size_t>(Bc) * F);
    c_counts.resize(Bc);
    QuerySource q;
    q.host = queries + static_cast<size_t>(c0) * ix->dim;
    float ms = 0.f;
    // the candidates: rbk_index_search_each_f64 on the route of the chunk's largest fetch_k
    st = F <= RBK_MAX_K_FETCH
             ? search_locked(ix, q, 8, Bc, F, -INFINITY, nullptr, nullptr, nullptr, c_slots.data(), c_scores.data(),
                             c_counts.data(), &ms, fetch_k + c0, min_score + c0)
             : large_locked(ix, q, Bc, F, -INFINITY, c_slots.data(), c_scores.data(), c_counts.data(), &ms,
                            fetch_k + c0, min_score + c0);
    if (st != RBK_OK) return st;
    const size_t o = static_cast<size_t>(c0) * K;
    st = mmr_select_locked(ix, Bc, F, c_slots.data(), c_scores.data(), c_counts.data(), k + c0, lambda_mult + c0, K,
                           stage, /*check_dead=*/true, out_slots + o, out_scores + o, out_counts + c0, &ms);
    if (st != RBK_OK) return st;
    if (kernel_ms_out) *kernel_ms_out += ms;
  }
  ix->stats.searches = searches;
  return RBK_OK;
}

rbk_status rbk_index_similar_pairs_f64(rbk_index* ix, double min_score, int64_t first_slot, int64_t max_pairs,
                                       int64_t* out_a, int64_t* out_b, double* out_scores, int64_t* n_out,
                                       int64_t* next_slot, float* kernel_ms_out) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  if (ix->slot.block != 0) return fail(RBK_EINVAL, "a group member answers through rbk_group_similar_pairs_f64");
  std::lock_guard<std::mutex> lk(ix->mu);
  rbk_status st = check_pairs_args(ix->slot.base, ix->n_rows, min_score, first_slot, max_pairs, out_a, out_b,
                                   out_scores, n_out, next_slot);
  if (st != RBK_OK) return st;
  DeviceGuard dg(ix->device);
  std::vector<int64_t> rows;
  auto load = [&](int64_t a0, int Q) {
    rows.resize(Q);
    for (int q = 0; q < Q; ++q) rows[q] = a0 - ix->slot.base + q;
    return gather_queries(ix, rows.data(), Q);   // a tombstoned row becomes a query of zeros: no pairs
  };
  return similar_pairs_run({ix}, ix->slot.base + ix->n_rows, min_score, first_slot, max_pairs, load, out_a, out_b,
                           out_scores, n_out, next_slot, kernel_ms_out);
}

rbk_status rbk_index_exact_scores_f64(rbk_index* ix, const double* queries, int32_t B, int32_t query_dim,
                                      double* out_scores) {
  if (!ix) return fail(RBK_EINVAL, "null index");
  if (B < 0 || (B > 0 && (!queries || !out_scores))) return fail(RBK_EINVAL, "bad argument");
  if (query_dim != ix->dim) return fail(RBK_EDIM, "Vectors must have the same length");  // embedder.ts:170
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  if (B == 0 || ix->n_rows == 0) return RBK_OK;
  rbk_status st = ensure_query_scratch(ix, B, 8);
  if (st != RBK_OK) return st;
  const size_t n = static_cast<size_t>(B) * ix->n_rows;
  CK(ix->o_scores.ensure(n));
  CK(cudaMemcpyAsync(ix->q_raw.p, queries, static_cast<size_t>(B) * ix->dim * 8, cudaMemcpyHostToDevice, ix->stream));
  // the prep kernel gives the f64 copy and the reference's normA; its scan-side outputs are unused here
  CK(launch_prep_queries(ix->q_raw.p, 0, B, ix->dim, ix->dpad, -INFINITY, nullptr, query_buffers(ix, 0), ix->stream,
                         /*with_norm2=*/true, nullptr, 0, 0));
  CK(launch_exact_scores(ix->rows, ix->rows_x, ix->x_elem, ix->norm2, ix->dead_bits, ix->n_rows, ix->dim, ix->dpad, ix->q_f64.p,
                         ix->q_norm2.p, B, ix->o_scores.p, ix->stream));
  ix->stats.kernel_launches += 2;
  CK(cudaMemcpyAsync(out_scores, ix->o_scores.p, n * 8, cudaMemcpyDeviceToHost, ix->stream));
  CK(cudaStreamSynchronize(ix->stream));
  return RBK_OK;
}

rbk_status rbk_index_search_device_async(rbk_index* ix, const void* dev_queries_f32, int32_t B, int32_t k_fetch,
                                         double min_score, void* dev_out_slots, void* dev_out_scores,
                                         void* dev_out_counts, void* dev_out_flags) {
  if (B > 0 && (!dev_queries_f32 || !dev_out_slots || !dev_out_scores || !dev_out_counts || !dev_out_flags))
    return fail(RBK_EINVAL, "null device pointer");
  rbk_status st = check_search_args(ix, B, true, ix ? ix->dim : 0, k_fetch, min_score);
  if (st != RBK_OK) return st;
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  if (B == 0) return RBK_OK;
  st = ensure_query_scratch(ix, B, 4);
  if (st != RBK_OK) return st;
  return enqueue_search(ix, dev_queries_f32, 1, B, k_fetch, min_score, static_cast<long long*>(dev_out_slots),
                        static_cast<double*>(dev_out_scores), static_cast<int*>(dev_out_counts),
                        static_cast<int*>(dev_out_flags));
}

rbk_status rbk_merge_topk_device(int32_t device, void* cuda_stream, int32_t G, int32_t B, int32_t k_fetch,
                                 const void* dev_slots, const void* dev_scores, const void* dev_counts,
                                 void* dev_out_slots, void* dev_out_scores, void* dev_out_counts) {
  if (G < 1 || B < 0 || k_fetch < 1) return fail(RBK_EINVAL, "bad merge shape");
  if (B == 0) return RBK_OK;
  if (!dev_slots || !dev_scores || !dev_counts || !dev_out_slots || !dev_out_scores || !dev_out_counts)
    return fail(RBK_EINVAL, "null device pointer");
  DeviceGuard dg(device);
  const size_t nk = static_cast<size_t>(B) * k_fetch;
  CK(launch_merge_shards(G, B, k_fetch, dev_slots, dev_scores, dev_counts, nullptr, nk * 8, nk * 8,
                         static_cast<size_t>(B) * 4, 0, static_cast<long long*>(dev_out_slots),
                         static_cast<double*>(dev_out_scores), static_cast<int*>(dev_out_counts), nullptr,
                         static_cast<cudaStream_t>(cuda_stream)));
  return RBK_OK;
}

int64_t rbk_packed_block_bytes(int32_t B, int32_t k_fetch) { return ResultBlock(B, k_fetch).bytes; }
int64_t rbk_packed_flags_offset(int32_t B, int32_t k_fetch) { return ResultBlock(B, k_fetch).off_flags; }

rbk_status rbk_merge_topk_packed_device(int32_t device, void* cuda_stream, int32_t G, int32_t B, int32_t k_fetch,
                                        const void* dev_blocks, void* dev_out_slots, void* dev_out_scores,
                                        void* dev_out_counts, void* dev_out_flags) {
  if (G < 1 || B < 0 || k_fetch < 1) return fail(RBK_EINVAL, "bad merge shape");
  if (B == 0) return RBK_OK;
  if (!dev_blocks || !dev_out_slots || !dev_out_scores || !dev_out_counts)
    return fail(RBK_EINVAL, "null device pointer");
  DeviceGuard dg(device);
  const ResultBlock L(B, k_fetch);
  const char* base = static_cast<const char*>(dev_blocks);
  CK(launch_merge_shards(G, B, k_fetch, base, base + L.off_scores, base + L.off_counts,
                         dev_out_flags ? base + L.off_flags : nullptr, L.bytes, L.bytes, L.bytes, L.bytes,
                         static_cast<long long*>(dev_out_slots), static_cast<double*>(dev_out_scores),
                         static_cast<int*>(dev_out_counts), static_cast<int*>(dev_out_flags),
                         static_cast<cudaStream_t>(cuda_stream)));
  return RBK_OK;
}

rbk_status rbk_index_stats(rbk_index* ix, rbk_stats* out) {
  if (!ix || !out) return fail(RBK_EINVAL, "null argument");
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  resolve_scan_events(ix, false);   // fold in every scan that has finished; never blocks
  *out = ix->stats;
  return RBK_OK;
}

rbk_status rbk_index_debug_scores_f32(rbk_index* ix, const float* queries, int32_t B, float* out_scores) {
  if (!ix || !queries || !out_scores || B < 1) return fail(RBK_EINVAL, "bad argument");
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  if (ix->n_rows == 0) return RBK_OK;
  rbk_status st = ensure_query_scratch(ix, B, 4);
  if (st != RBK_OK) return st;
  const size_t n = static_cast<size_t>(B) * ix->n_rows;
  CK(ix->dbg.ensure(n));
  CK(cudaMemsetAsync(ix->dbg.p, 0xFF, n * 4, ix->stream));
  CK(cudaMemcpyAsync(ix->q_raw.p, queries, static_cast<size_t>(B) * ix->dim * 4, cudaMemcpyHostToDevice, ix->stream));
  st = run_scan(ix, ix->q_raw.p, 1, B, 16, -INFINITY, nullptr, nullptr, nullptr, nullptr, ix->dbg.p);
  if (st != RBK_OK) return st;
  std::vector<float> invq(B);
  CK(cudaMemcpyAsync(out_scores, ix->dbg.p, n * 4, cudaMemcpyDeviceToHost, ix->stream));
  CK(cudaMemcpyAsync(invq.data(), ix->q_inv_norm.p, sizeof(float) * B, cudaMemcpyDeviceToHost, ix->stream));
  CK(cudaStreamSynchronize(ix->stream));
  for (int b = 0; b < B; ++b)
    for (int64_t r = 0; r < ix->n_rows; ++r) out_scores[static_cast<size_t>(b) * ix->n_rows + r] *= invq[b];
  return RBK_OK;
}

}  // extern "C"
