// rbk_scan.cu — K1: fused  Q x C^T (wgmma, bf16 -> fp32 in registers)  +  row-norm scaling
//               +  per-query running top-k' selection in the epilogue.
//
// Replaces the hot loop of VectorStore.search (reference src/knowledge/store/
// vector-store.ts:207-215 calling cosineSimilarity, src/knowledge/indexer/
// embedder.ts:168-184) for a whole batch of queries at once.  The score matrix never
// reaches HBM: the tile's accumulators go to shared memory, where each epilogue thread
// owns one query (one row), compares its 256 scores with that query's running threshold
// and appends the rare survivors to a small per-(CTA, query) candidate list.
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
// Pipelines: smem ring full/empty (TMA <-> wgmma); one score buffer full/empty (wgmma <->
//   epilogue).  The accumulators live in registers while the next tile is multiplied, so the
//   epilogue of tile i overlaps the wgmma of tile i+1 with a single smem score buffer.
#include "rbk_epilogue.cuh"
#include "rbk_internal.h"
#include "rbk_ptx.cuh"

namespace rbk {

namespace {

constexpr int kABytes = kBlockM * kBlockK * 2;      // 8 KiB   query k-slab
constexpr int kBBytes = kBlockN * kBlockK * 2;      // 16 KiB  corpus k-slab
constexpr int kStageBytes = kABytes + kBBytes;      // 24 KiB
constexpr int kMmaThreads = 256;                    // warpgroups 1-2
constexpr int kScoreBytes = kBlockM * kScorePitch * 4;
static_assert(kScanThreads == 128 + kMmaThreads, "warp roles");

struct SmemTail {
  float invc[2][kBlockN];  // 1/||c|| of the tile's rows, double-buffered by tile parity
  unsigned long long full[kStages];
  unsigned long long empty[kStages];
  unsigned long long sc_full;
  unsigned long long sc_empty;
};

// Accumulator fragment of one warpgroup thread -> score rows (see wgmma_m64n256k16_bf16).
__device__ __forceinline__ void store_accumulators(float* scores, const float (&d)[128], int wg, int warp, int lane) {
  const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  float* r0 = scores + row * kScorePitch + 2 * (lane & 3);
  float* r1 = r0 + 8 * kScorePitch;
#pragma unroll
  for (int j = 0; j < kBlockN / 8; ++j) {
    *reinterpret_cast<float2*>(r0 + 8 * j) = make_float2(d[4 * j + 0], d[4 * j + 1]);
    *reinterpret_cast<float2*>(r1 + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

__global__ void __launch_bounds__(kScanThreads, 1)
scan_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_c,
            const ScanParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);  // swizzled TMA boxes want 1024-B alignment
  float* scores = reinterpret_cast<float*>(smem + kStages * kStageBytes);
  SmemTail* tail = reinterpret_cast<SmemTail*>(smem + kStages * kStageBytes + kScoreBytes);
  const uint32_t smem_base = smem_u32(smem);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wgroup = warp >> 2;
  const int qb = blockIdx.x % p.QB;
  const int r = blockIdx.x / p.QB;
  const int t0 = static_cast<int>(static_cast<long long>(p.n_tiles) * r / p.R);
  const int t1 = static_cast<int>(static_cast<long long>(p.n_tiles) * (r + 1) / p.R);
  const int n_ks = p.dpad / kBlockK;

  if (threadIdx.x == 128) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_c);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(smem_u32(&tail->full[s]), 1);
      mbar_init(smem_u32(&tail->empty[s]), 2);   // one arrive per wgmma warpgroup
    }
    mbar_init(smem_u32(&tail->sc_full), kMmaThreads);
    mbar_init(smem_u32(&tail->sc_empty), 128);   // every epilogue thread
    fence_barrier_init();
  }
  __syncthreads();

  if (wgroup == 0) {
    // ===================== epilogue: thread <-> query =====================
    run_epilogue(p, tail->invc, &tail->sc_full, &tail->sc_empty, scores, qb, r, t0, t1, threadIdx.x, lane);
    return;
  }

  // ===================== wgmma: warpgroup wg <-> queries 64 wg .. 64 wg + 63 =====================
  const int wg = wgroup - 1;
  const bool leader = (threadIdx.x & 127) == 0;
  const bool producer = warp == 4;
  const int n_steps = (t1 - t0) * n_ks;   // k-steps of the whole unit; step j uses ring slot j % kStages
  volatile int* prog = p.progress + r * p.QB;
  // Load step j into its slot once both warpgroups have released the slot's previous use (whole warp).
  auto issue = [&](int j) {
    if (j >= n_steps) return;
    const int s = j % kStages;
    const int tile = t0 + j / n_ks, ks = j % n_ks;
    mbar_wait(smem_u32(&tail->empty[s]), static_cast<uint32_t>((j / kStages) & 1) ^ 1u);
    if (ks == 0 && lane == 0) lockstep_pace(prog, p.QB, qb, tile - t0, p.max_lead_tiles);
    __syncwarp();
    const uint32_t full = smem_u32(&tail->full[s]);
    const uint32_t a_dst = smem_base + s * kStageBytes;
    if (elect_one()) {
      mbar_arrive_expect_tx(full, kStageBytes);
      tma_load_2d(a_dst, &tmap_q, full, ks * kBlockK, qb * kBlockM);
      tma_load_2d(a_dst + kABytes, &tmap_c, full, ks * kBlockK, tile * kBlockN);
    }
    __syncwarp();
  };
  // a step's slot is released (and refilled kStages steps ahead) once its wgmma group has retired
  auto release = [&](int j) {
    if (leader) mbar_arrive(smem_u32(&tail->empty[j % kStages]));
    if (producer) issue(j + kStages);
  };
  if (producer)
    for (int j = 0; j < kStages; ++j) issue(j);
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  int j = 0;
  for (int tile = t0; tile < t1; ++tile) {
    for (int ks = 0; ks < n_ks; ++ks, ++j) {
      const int s = j % kStages;
      mbar_wait(smem_u32(&tail->full[s]), static_cast<uint32_t>((j / kStages) & 1));
      const uint32_t st = smem_base + s * kStageBytes;
      const uint64_t adesc = make_sw64_kmajor_desc(st + wg * (64 * kBlockK * 2));
      const uint64_t bdesc = make_sw64_kmajor_desc(st + kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)   // +32 bytes per k-step = +2 in the 16-byte address field
        wgmma_m64n256k16_bf16(acc, adesc + static_cast<uint64_t>(2 * k), bdesc + static_cast<uint64_t>(2 * k),
                              (ks | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>(acc);   // the previous step's group has retired
      if (ks > 0) release(j - 1);
    }
    wgmma_wait<0>(acc);
    release(j - 1);
    // the epilogue has finished reading the previous tile's scores
    mbar_wait(smem_u32(&tail->sc_empty), static_cast<uint32_t>((tile - t0) & 1) ^ 1u);
    store_accumulators(scores, acc, wg, warp, lane);
    mbar_arrive(smem_u32(&tail->sc_full));
  }
  if (producer && lane == 0 && p.QB > 1) prog[qb] = 0x7FFFFFFF;  // done: never hold a peer back
}

}  // namespace

cudaError_t launch_scan(const CUtensorMap& tmap_q, const CUtensorMap& tmap_c, const ScanParams& p,
                        cudaStream_t stream) {
  const size_t smem = static_cast<size_t>(kStages) * kStageBytes + kScoreBytes + sizeof(SmemTail) + 1024;
  // per-device attribute; cheap enough to set on every launch
  cudaError_t e = cudaFuncSetAttribute(scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  scan_kernel<<<p.QB * p.R, kScanThreads, smem, stream>>>(tmap_q, tmap_c, p);
  return cudaGetLastError();
}

}  // namespace rbk
