// rbk_scan_kernel.cuh — the fused scan kernel (see rbk_scan.cu for what it does), compiled once per corpus element
// type: rbk_scan.cu includes it with RBK_SCAN_F16 = 0 (bf16 rows, every index by default), rbk_scan_f16.cu with
// RBK_SCAN_F16 = 1 (fp16 rows, RBK_INDEX_SCAN_F16).  The two kernels differ only in the HGMMA operand type; the tiles,
// descriptors, swizzle, fragment layout and epilogues are the same bytes.  Everything here is in an anonymous
// namespace, so each translation unit gets its own kernels and the includer defines the launchers.
// The RBK_SCAN_CYCLE_STATS probe lives in the bf16 translation unit only.
#pragma once
#ifndef RBK_SCAN_F16
#error "define RBK_SCAN_F16 (0: bf16 operands, 1: fp16 operands) before including rbk_scan_kernel.cuh"
#endif
#if defined(RBK_SCAN_CYCLE_STATS) && !RBK_SCAN_F16
#define RBK_SCAN_PROBE 1
#else
#define RBK_SCAN_PROBE 0
#endif

#include "rbk_epilogue.cuh"
#include "rbk_internal.h"
#include "rbk_ptx.cuh"

namespace rbk {

namespace {

constexpr int kABytes = kBlockM * kBlockK * 2;      // 16 KiB  query k-slab
constexpr int kBBytes = kBlockN * kBlockK * 2;      // 32 KiB  corpus k-slab
constexpr int kStageBytes = kABytes + kBBytes;      // 48 KiB
constexpr int kMmaThreads = 256;                    // warpgroups 1-2
constexpr int kStagingBytes = 2 * kStageRows * kScorePitch * 4;   // one staging buffer per wgmma warpgroup
static_assert(kScanThreads == 128 + kMmaThreads, "warp roles");
static_assert(2 * kStageRows <= kBlockM, "a round never holds more rows than a warpgroup has queries");

struct SmemTail {
  float invc[2][2][kBlockN];   // [wgmma warpgroup][tile parity] 1/||c|| of the tile's rows (bulk copies)
  float thr[kBlockM];          // per-query threshold the epilogue thread last published (only rises)
  StageHeader hdr[2];
  uint16_t wmask[2][2][4];     // [warpgroup][tile parity][warp] queries of the warp that pass the prefilter
  unsigned long long full[kStages];
  uint32_t released[kStages];   // releases of the slot so far, two per use (one per wgmma warpgroup)
#if RBK_SCAN_PROBE
  uint32_t issue_clk[kStages];  // SM clock at the slot's last TMA issue
#endif
  unsigned long long invc_full[2][2];
  unsigned long long st_full[2];
  unsigned long long st_empty[2];
};
constexpr size_t kScanSmemBytes = static_cast<size_t>(kStages) * kStageBytes + kStagingBytes + sizeof(SmemTail) + 1024;
static_assert(kScanSmemBytes <= 227 * 1024, "scan kernel shared memory exceeds the sm_90 per-block limit");

// The tensor-core step of the main loop, in the corpus's element type.
__device__ __forceinline__ void scan_mma(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
#if RBK_SCAN_F16
  wgmma_m64n256k16_f16(d, desc_a, desc_b, accumulate);
#else
  wgmma_m64n256k16_bf16(d, desc_a, desc_b, accumulate);
#endif
}

// One row of a wgmma warpgroup thread's accumulator fragment (h = 0: d[4j + 0..1], h = 1: d[4j + 2..3]; see
// wgmma_m64n256k16_bf16) -> its columns of a staged row.
__device__ __forceinline__ void store_row(float* dst, const float (&d)[128], int h, int lane) {
  float* r = dst + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < kBlockN / 8; ++j)
    *reinterpret_cast<float2*>(r + 8 * j) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
}

// Ballot of a row predicate voted alike by the 4 lanes of each quad -> 8 bits, bit i = quad i.
__device__ __forceinline__ uint32_t quad_bits(uint32_t b) {
  b &= 0x11111111u;
  b = (b | (b >> 3)) & 0x03030303u;
  b = (b | (b >> 6)) & 0x000F000Fu;
  return (b | (b >> 12)) & 0xFFu;
}

// Development probe (RBK_SCAN_CYCLE_STATS): where a wgmma warpgroup's cycles go.  Its leader thread adds SM-clock
// deltas into buckets, summed over the launch per warpgroup:
//   full     waiting on a ring slot's `full` barrier;
//   mma      fence, HGMMA issue and wait_group until the previous group has retired (tensor work);
//   handoff  from wait_group returning to the end of the slot release: pacing (warpgroup 1), the release count and,
//            in the warpgroup that released the slot last, the TMA issue of its refill.  Nobody waits here for the
//            other warpgroup;
//   pace     the part of handoff spent on lockstep (warpgroup 1 only: its first warp paces the CTA);
//   refill   the part of handoff its leader spent issuing refills, `refills` of them;
//   tile_end wait_group 0, the last release, the prefilter, the st_empty waits and the row staging;
//   fetch    not a lap: over the `fetch_waits` full waits that found the barrier still pending, cycles from the slot's
//            TMA issue (either warpgroup's) to the wait's return, i.e. how long a copy that is waited for takes.
// The laps are contiguous, so full + mma + handoff + tile_end is the whole main loop.  The kernel only adds; the host
// reads and clears the sums with rbk_scan_cycle_stats (no printf: a call inside the kernel makes ptxas serialize the
// wgmma pipeline, and the probe would time another kernel).  The probe's registers cost the top-k' instantiation
// about 20 bytes of spills.  Without the macro CycleProbe is empty and compiles to nothing.
enum CycleBucket { kCycFull, kCycMma, kCycHandoff, kCycPace, kCycRefill, kCycTileEnd, kCycFetch, kCycBuckets };
constexpr int kCycCounters = 4;   // after the buckets: tiles, units, fetch_waits, refills
#if RBK_SCAN_PROBE
__device__ unsigned long long g_cycle_stats[3][2][kCycBuckets + kCycCounters];   // [mode][warpgroup][...]
__device__ __forceinline__ uint32_t sm_clock() {
  uint32_t c;
  asm volatile("mov.u32 %0, %%clock;" : "=r"(c)::"memory");
  return c;
}
struct CycleProbe {
  uint32_t t = 0, c[kCycBuckets] = {}, fetch_waits = 0, refills = 0;
  __device__ __forceinline__ void mark() { t = sm_clock(); }
  __device__ __forceinline__ void lap(int b) {   // t .. now into bucket b; now becomes t
    const uint32_t n = sm_clock();
    c[b] += n - t;
    t = n;
  }
  __device__ __forceinline__ void add_since(int b, uint32_t t0) { c[b] += sm_clock() - t0; }
  __device__ __forceinline__ void refilled(uint32_t t0) {
    add_since(kCycRefill, t0);
    ++refills;
  }
  __device__ __forceinline__ void fetched(uint32_t issue_clk) {   // a full wait that blocked has returned
    add_since(kCycFetch, issue_clk);
    ++fetch_waits;
  }
  __device__ __forceinline__ static uint32_t now() { return sm_clock(); }
};
#else
struct CycleProbe {
  __device__ __forceinline__ void mark() {}
  __device__ __forceinline__ void lap(int) {}
  __device__ __forceinline__ void add_since(int, uint32_t) {}
  __device__ __forceinline__ void refilled(uint32_t) {}
  __device__ __forceinline__ static uint32_t now() { return 0u; }
};
#endif

// kMode 0: top-k' candidate lists (P = ScanParams); kScanCount / kScanEmit: the large-k passes (P = LargeScanParams)
template <int kMode, typename P>
__global__ void __launch_bounds__(kScanThreads, 1)
scan_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_c,
            const P p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);  // swizzled TMA boxes want 1024-B alignment
  float* staging = reinterpret_cast<float*>(smem + kStages * kStageBytes);
  SmemTail* tail = reinterpret_cast<SmemTail*>(smem + kStages * kStageBytes + kStagingBytes);
  const uint32_t smem_base = smem_u32(smem);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wgroup = warp >> 2;
  const int qb = blockIdx.x % p.QB;
  const int r = blockIdx.x / p.QB;
  const int t0 = static_cast<int>(static_cast<long long>(p.n_tiles) * r / p.R);
  const int t1 = static_cast<int>(static_cast<long long>(p.n_tiles) * (r + 1) / p.R);
  const int n_ks = p.dpad / kBlockK;

  if (threadIdx.x < kBlockM) tail->thr[threadIdx.x] = -INFINITY;
  if (threadIdx.x == 128) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_c);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(smem_u32(&tail->full[s]), 1);
      tail->released[s] = 0u;
    }
    for (int w = 0; w < 2; ++w) {
      mbar_init(smem_u32(&tail->invc_full[w][0]), 1);
      mbar_init(smem_u32(&tail->invc_full[w][1]), 1);
      mbar_init(smem_u32(&tail->st_full[w]), 128);   // every thread of the wgmma warpgroup
      mbar_init(smem_u32(&tail->st_empty[w]), 64);   // the epilogue threads of its 64 queries
    }
    fence_barrier_init();
  }
  __syncthreads();

  // The launch bound gives every thread 168 registers.  The wgmma warpgroups carry 128 accumulators and the prefilter;
  // the epilogue needs less: 128 x kEpiRegs + 256 x kMmaRegs = 384 x 168.
  constexpr uint32_t kEpiRegs = 152, kMmaRegs = 176;
  static_assert(128 * kEpiRegs + kMmaThreads * kMmaRegs <= kScanThreads * 168, "register split");
  if (wgroup == 0) {
    // ===================== epilogue: thread <-> query =====================
    setmaxnreg_dec<kEpiRegs>();
    const int h = threadIdx.x >> 6;   // the wgmma warpgroup that holds this query's accumulators
    const StageLink sl{staging + h * kStageRows * kScorePitch, &tail->hdr[h], &tail->st_full[h], &tail->st_empty[h],
                       &tail->thr[threadIdx.x]};
    if constexpr (kMode == 0)
      run_epilogue(p, sl, qb, r, t0, t1, threadIdx.x, lane);
    else if constexpr (kMode == kScanCount)
      run_count_epilogue(p, sl, qb, t0, t1, threadIdx.x);
    else
      run_emit_epilogue(p, sl, qb, t0, t1, threadIdx.x);
    return;
  }

  // ===================== wgmma: warpgroup wg <-> queries 64 wg .. 64 wg + 63 =====================
  setmaxnreg_inc<kMmaRegs>();
  const int wg = wgroup - 1;
  const bool leader = (threadIdx.x & 127) == 0;
  const int n_iter = t1 - t0;
  volatile int* prog = p.progress + r * p.QB;
  CycleProbe probe;
  // Load k-slab ks of tile t0 + it into ring slot s (one thread).
  auto issue = [&](int s, int it, int ks) {
    const uint32_t issue0 = CycleProbe::now();
#if RBK_SCAN_PROBE
    tail->issue_clk[s] = issue0;
#endif
    const uint32_t full = smem_u32(&tail->full[s]);
    const uint32_t a_dst = smem_base + s * kStageBytes;
    mbar_arrive_expect_tx(full, kStageBytes);
    tma_load_2d(a_dst, &tmap_q, full, ks * kBlockK, qb * kBlockM);
    tma_load_2d(a_dst + kABytes, &tmap_c, full, ks * kBlockK, (t0 + it) * kBlockN);
    probe.refilled(issue0);
  };
  // Lockstep is the business of warpgroup 1's first warp: it holds back its own release of the slot that a paced
  // tile's first k-slab goes into, and with it the refill, whichever warpgroup issues that.  Its lanes read the
  // peers' progress two refills earlier (as early as the tile before when n_ks < 3), so the check itself waits for
  // no load.  seen starts as "nobody behind": the first check of a unit whose tiles are one k-slab is skipped.
  const bool pacer = warp == 4 && p.QB > 1;
  const bool peer = lane < p.QB && lane != qb;
  const int peek_ks = n_ks > 2 ? n_ks - 2 : 0;
  int seen = 0x7FFFFFFF;
  // The step that refills the slot released next: k-slab r_ks of tile t0 + r_it (kStages steps after the released one).
  int r_it = kStages / n_ks, r_ks = kStages % n_ks;
  // Slot s is released by a warpgroup once its wgmma group on it has retired.  The warpgroup that does so last
  // refills it there and then, from its leader thread, and nobody waits for the other: the leaders count releases in
  // released[s], two per use of the slot, so the one whose add returns an odd count is the second.  Ordering: the
  // leader's wgmma_wait has retired its warpgroup's reads of the slot before its add; the add is acq_rel at CTA scope,
  // so the second leader's add has acquired the first one's, and its TMA issue follows in program order - the chain
  // an `empty` mbarrier (arrive, arrive, wait, issue) would give.  Measured against that mbarrier kept for the
  // ordering beside a relaxed add (arrive, add, and a wait by the second), this is the faster of the two (DESIGN §7).
  // A warpgroup that runs ahead stops at a `full` wait.
  auto release = [&](int s) {
    // every other tile: pacing every tile costs ~10 % on short kernels
    if (pacer && r_ks == 0 && (r_it & 1) == 0 && r_it < n_iter) {
      const uint32_t pace0 = CycleProbe::now();
      lockstep_pace(prog, qb, r_it, p.max_lead_tiles, lane, peer, seen);
      probe.add_since(kCycPace, pace0);
    }
    if (leader && (smem_inc_acq_rel(smem_u32(&tail->released[s])) & 1u) != 0u && r_it < n_iter) issue(s, r_it, r_ks);
    // after the add: its release fence would wait for the load
    if (pacer && r_ks == peek_ks && (r_it & 1) != 0) lockstep_peek(prog, lane, peer, seen);
    if (++r_ks == n_ks) {
      r_ks = 0;
      ++r_it;
    }
  };
  // 1/||c|| of tile t0 + i for this warpgroup's prefilter, into buffer i & 1
  auto load_invc = [&](int i) {
    if (!leader || i >= n_iter) return;
    const uint32_t bar = smem_u32(&tail->invc_full[wg][i & 1]);
    mbar_arrive_expect_tx(bar, kBlockN * 4);
    bulk_load(smem_u32(tail->invc[wg][i & 1]), p.inv_norm_c + static_cast<size_t>(t0 + i) * kBlockN, kBlockN * 4, bar);
  };
  if (leader && wg == 0)
    for (int j = 0; j < kStages && j / n_ks < n_iter; ++j) issue(j, j / n_ks, j % n_ks);
  load_invc(0);
  load_invc(1);
  // this thread's accumulator rows: query qw0 (d[4j + 0..1]) and qw1 (d[4j + 2..3]) of the warpgroup's 64
  const int qw0 = (warp & 3) * 16 + (lane >> 2);
  const int qw1 = qw0 + 8;
  const volatile float* thr = tail->thr + wg * 64;
  float* stage = staging + wg * kStageRows * kScorePitch;
  const uint32_t st_full = smem_u32(&tail->st_full[wg]), st_empty = smem_u32(&tail->st_empty[wg]);
  uint32_t rounds = 0;
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  int j = 0;
  probe.mark();
  for (int i = 0; i < n_iter; ++i) {
    for (int ks = 0; ks < n_ks; ++ks, ++j) {
      const int s = j % kStages;
      const uint32_t full = smem_u32(&tail->full[s]), parity = static_cast<uint32_t>((j / kStages) & 1);
#if RBK_SCAN_PROBE
      const bool blocked = leader && !mbar_try_wait(full, parity);
#endif
      mbar_wait(full, parity);
#if RBK_SCAN_PROBE
      if (blocked) probe.fetched(tail->issue_clk[s]);
#endif
      probe.lap(kCycFull);
      const uint32_t st = smem_base + s * kStageBytes;
      const uint64_t adesc = make_sw128_kmajor_desc(st + wg * (64 * kBlockK * 2));
      const uint64_t bdesc = make_sw128_kmajor_desc(st + kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)   // +32 bytes per k-step = +2 in the 16-byte address field
        scan_mma(acc, adesc + static_cast<uint64_t>(2 * k), bdesc + static_cast<uint64_t>(2 * k), (ks | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>(acc);   // the previous step's group has retired
      probe.lap(kCycMma);
      if (ks > 0) release((j - 1) % kStages);
      probe.lap(kCycHandoff);
    }
    wgmma_wait<0>(acc);
    release((j - 1) % kStages);

    // Prefilter: scores = accumulator * 1/||c|| (the very multiply the epilogue used to do), then each row's maximum
    // against the threshold its epilogue thread last published.  fmaxf drops the NaN of dead rows.
    mbar_wait(smem_u32(&tail->invc_full[wg][i & 1]), static_cast<uint32_t>((i >> 1) & 1));
    const float* invc = tail->invc[wg][i & 1] + 2 * (lane & 3);
    float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
    for (int c = 0; c < kBlockN / 8; ++c) {
      const float2 w = *reinterpret_cast<const float2*>(invc + 8 * c);
      acc[4 * c + 0] *= w.x;
      acc[4 * c + 1] *= w.y;
      acc[4 * c + 2] *= w.x;
      acc[4 * c + 3] *= w.y;
      m0 = fmaxf(m0, fmaxf(acc[4 * c + 0], acc[4 * c + 1]));
      m1 = fmaxf(m1, fmaxf(acc[4 * c + 2], acc[4 * c + 3]));
    }
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {   // the 4 lanes of a quad hold the same two rows
      m0 = fmaxf(m0, __shfl_xor_sync(0xFFFFFFFFu, m0, o));
      m1 = fmaxf(m1, __shfl_xor_sync(0xFFFFFFFFu, m1, o));
    }
    bool pass0, pass1;
    if constexpr (kMode == 0) {
      // the seeding pass reads every score of a unit's first tile; debug scores want every score
      const bool all = i == 0 || p.dbg_scores != nullptr;
      pass0 = all || m0 > thr[qw0];
      pass1 = all || m1 > thr[qw1];
    } else {
      pass0 = m0 >= thr[qw0];
      pass1 = m1 >= thr[qw1];
    }
    const uint32_t wbits = quad_bits(__ballot_sync(0xFFFFFFFFu, pass0)) |
                           (quad_bits(__ballot_sync(0xFFFFFFFFu, pass1)) << 8);
    if (lane == 0) tail->wmask[wg][i & 1][warp & 3] = static_cast<uint16_t>(wbits);
    named_bar_sync(2 + wg, 128);   // also: every thread of the warpgroup is done with invc[i & 1]
    load_invc(i + 2);
    const uint16_t* wm = tail->wmask[wg][i & 1];
    unsigned long long pending = static_cast<unsigned long long>(wm[0]) | static_cast<unsigned long long>(wm[1]) << 16 |
                                 static_cast<unsigned long long>(wm[2]) << 32 | static_cast<unsigned long long>(wm[3]) << 48;

    // Hand the passing rows over, at most kStageRows per round; a tile without any is one round with no rows.
    do {
      unsigned long long cur = pending;
      if (__popcll(pending) > kStageRows) {
        unsigned long long rest = pending;
        for (int k = 0; k < kStageRows; ++k) rest &= rest - 1ull;
        cur = pending ^ rest;
      }
      pending ^= cur;
      mbar_wait(st_empty, (rounds & 1u) ^ 1u);   // the epilogue has finished the previous round
      if ((cur >> qw0) & 1ull) store_row(stage + __popcll(cur & ((1ull << qw0) - 1ull)) * kScorePitch, acc, 0, lane);
      if ((cur >> qw1) & 1ull) store_row(stage + __popcll(cur & ((1ull << qw1) - 1ull)) * kScorePitch, acc, 1, lane);
      if (leader) {
        tail->hdr[wg].mask = cur;
        tail->hdr[wg].last = pending == 0ull;
      }
      mbar_arrive(st_full);
      ++rounds;
    } while (pending != 0ull);
    probe.lap(kCycTileEnd);
  }
  if (pacer && lane == 0) prog[qb] = 0x7FFFFFFF;  // done: never hold a peer back
#if RBK_SCAN_PROBE
  if (leader) {   // the host reads the sums (rbk_scan_cycle_stats): a call here would serialize the wgmma pipeline
    for (int b = 0; b < kCycBuckets; ++b)
      atomicAdd(&g_cycle_stats[kMode][wg][b], static_cast<unsigned long long>(probe.c[b]));
    atomicAdd(&g_cycle_stats[kMode][wg][kCycBuckets], static_cast<unsigned long long>(n_iter));
    atomicAdd(&g_cycle_stats[kMode][wg][kCycBuckets + 1], 1ull);
    atomicAdd(&g_cycle_stats[kMode][wg][kCycBuckets + 2], static_cast<unsigned long long>(probe.fetch_waits));
    atomicAdd(&g_cycle_stats[kMode][wg][kCycBuckets + 3], static_cast<unsigned long long>(probe.refills));
  }
#endif
}

template <int kMode, typename P>
cudaError_t launch_scan_mode(const CUtensorMap& tmap_q, const CUtensorMap& tmap_c, const P& p, cudaStream_t stream) {
  // per-device attribute; cheap enough to set on every launch
  cudaError_t e = cudaFuncSetAttribute(scan_kernel<kMode, P>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)kScanSmemBytes);
  if (e != cudaSuccess) return e;
  scan_kernel<kMode, P><<<p.QB * p.R, kScanThreads, kScanSmemBytes, stream>>>(tmap_q, tmap_c, p);
  return cudaGetLastError();
}

}  // namespace
}  // namespace rbk
