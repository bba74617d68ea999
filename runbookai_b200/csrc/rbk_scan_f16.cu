// rbk_scan_f16.cu — the fused scan of rbk_scan.cu with fp16 operands, for indexes created with RBK_INDEX_SCAN_F16.
//
// Such an index stores every row, and every query, as fp16 scaled by a per-row power of two (DESIGN.md §3): 11
// significant bits instead of bf16's 8, at the same 2 bytes per element, so the scan's error bound is several times
// tighter (DESIGN.md §6).  The kernel is the bf16 one with the HGMMA operand type changed
// (wgmma.mma_async ... f32.f16.f16); products of two fp16 values are exact in fp32, as products of two bf16 values
// are, and the accumulators, the prefilter and the epilogues are unchanged.  The cycle probe is not built here.
#define RBK_SCAN_F16 1
#include "rbk_scan_kernel.cuh"

namespace rbk {

cudaError_t launch_scan_f16(const CUtensorMap& tmap_q, const CUtensorMap& tmap_c, const ScanParams& p,
                            cudaStream_t stream) {
  return launch_scan_mode<0>(tmap_q, tmap_c, p, stream);
}

cudaError_t launch_scan_large_f16(const CUtensorMap& tmap_q, const CUtensorMap& tmap_c, const LargeScanParams& p,
                                  LargeScanMode mode, cudaStream_t stream) {
  if (mode == kScanCount) return launch_scan_mode<kScanCount>(tmap_q, tmap_c, p, stream);
  return launch_scan_mode<kScanEmit>(tmap_q, tmap_c, p, stream);
}

}  // namespace rbk
