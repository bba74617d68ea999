// rbk_scan.cu — K1: fused  Q x C^T (wgmma, bf16 -> fp32 in registers)  +  row-norm scaling
//               +  per-query running top-k' selection in the epilogue.
//
// Replaces the hot loop of VectorStore.search (reference src/knowledge/store/
// vector-store.ts:207-215 calling cosineSimilarity, src/knowledge/indexer/
// embedder.ts:168-184) for a whole batch of queries at once.  The score matrix never
// reaches HBM: the wgmma warpgroups scale their accumulators by 1/||c|| in registers and
// compare each row's maximum with the threshold its epilogue thread last published; only
// rows that can hold a survivor go to shared memory, where each epilogue thread owns one
// query (one row), filters its 256 scores and appends the survivors to a small
// per-(CTA, query) candidate list.
//
// Work decomposition (persistent CTAs, at most one per SM):
//   CTA c -> query block qb = c % QB (128 queries), corpus range r = c / QB.
//   CTAs that share r walk the same corpus tiles at the same pace, so a tile is pulled
//   from HBM once and served to the other query blocks from L2.
// Warp roles: warpgroup 0 = epilogue (thread <-> query), warpgroups 1 / 2 = wgmma (queries
//   0-63 / 64-127 of the block, all 256 rows of the tile); the first warp of warpgroup 1 also
//   refills the smem ring (TMA, elected lane) once both warpgroups have released a slot.  The
//   64 x 256 fp32 accumulator takes 128 registers per thread: with 12 warps (three per SM
//   sub-partition) the launch bound leaves 168, with a separate producer warp it would be 128.
// Pipelines: smem ring of 64-column stages, full/empty (TMA <-> wgmma); per wgmma warpgroup one
//   staging buffer of kStageRows rows, full/empty per round (wgmma -> epilogue; every tile is at
//   least one round, a tile with more passing rows than fit takes several).  The epilogue of
//   tile i overlaps the wgmma of tile i + 1.  Dropping a (query, tile) pair is safe because
//   thresholds only rise: see DESIGN.md §6.
//
// The kernel itself is in rbk_scan_kernel.cuh, shared with the fp16 scan of rbk_scan_f16.cu.
#define RBK_SCAN_F16 0
#include "rbk_scan_kernel.cuh"

namespace rbk {

cudaError_t launch_scan(const CUtensorMap& tmap_q, const CUtensorMap& tmap_c, const ScanParams& p,
                        cudaStream_t stream) {
  return launch_scan_mode<0>(tmap_q, tmap_c, p, stream);
}

cudaError_t launch_scan_large(const CUtensorMap& tmap_q, const CUtensorMap& tmap_c, const LargeScanParams& p,
                              LargeScanMode mode, cudaStream_t stream) {
  if (mode == kScanCount) return launch_scan_mode<kScanCount>(tmap_q, tmap_c, p, stream);
  return launch_scan_mode<kScanEmit>(tmap_q, tmap_c, p, stream);
}

}  // namespace rbk

#ifdef RBK_SCAN_CYCLE_STATS
// Probe builds only: waits for the current device, copies its cycle sums ([mode][warpgroup][full, mma, handoff, pace,
// refill, tile_end, fetch, tiles, units, fetch_waits, refills], 66 values) to out and clears them.  Returns the number
// of values, or -1 on a CUDA error.
extern "C" int rbk_scan_cycle_stats(unsigned long long* out) {
  constexpr int n = 3 * 2 * (rbk::kCycBuckets + rbk::kCycCounters);
  static const unsigned long long zero[n] = {};
  if (cudaDeviceSynchronize() != cudaSuccess ||
      cudaMemcpyFromSymbol(out, rbk::g_cycle_stats, sizeof(zero)) != cudaSuccess ||
      cudaMemcpyToSymbol(rbk::g_cycle_stats, zero, sizeof(zero)) != cudaSuccess)
    return -1;
  return n;
}
#endif
