// rbk_epilogue.cuh — per-query candidate filter shared by the scan kernels' epilogues.
//
// One epilogue thread owns one query.  It keeps a running threshold `thr` (raw domain:
// accumulator * 1/||c||) and appends the rare survivors to its (CTA, query) list.  The
// threshold comes from three sources, all of them LOWER bounds on the query's global k'-th
// best score, so dropping a row at or below it is always safe:
//   1. min_score - eps (prep kernel),
//   2. the k'-th best of the thread's own list after a compaction,
//   3. a global per-query histogram of the scores of ALL appended rows (every CTA adds to
//      it): the highest bin edge with >= k' rows at or above it.  This is what makes the
//      threshold track the true running k'-th best of the whole corpus instead of one
//      CTA's slice, so after the first few chunks almost nothing is appended any more.
#pragma once
#include "rbk_internal.h"
#include "rbk_ptx.cuh"

namespace rbk {

struct FilterState {
  float thr;       // raw-domain threshold
  float inv_q;     // 1/||bf16(q)||: raw -> approximate cosine
  float qn;        // ||bf16(q)||
  int tb;          // histogram bin whose lower edge produced thr (-1: none yet)
  int mb_cache;    // highest bin this thread already published to maxbin
  int cnt;         // entries in the list
  bool valid;
  bool nohist;     // appends are not counted in the histogram (second pass over a seeded tile)
  unsigned long long* list;
  unsigned int* hist_q;  // [kHistBins]
  int* maxbin_q;
};

__device__ __forceinline__ int score_bin(float a) {
  const int b = static_cast<int>((a + 1.0f) * (kHistBins * 0.5f));
  return min(max(b, 0), kHistBins - 1);
}
// Raw threshold such that every row counted in bins >= b has raw score > the result.
__device__ __forceinline__ float bin_edge_raw(int b, float qn) {
  const float edge = static_cast<float>(b) * (2.0f / kHistBins) - 1.0f - 1e-6f;  // cosine domain, nudged down
  const float r = edge * qn;
  return r - fabsf(r) * 1e-6f;
}

__device__ __forceinline__ void filter_init(FilterState& s, bool valid, float thr_init, float inv_q,
                                            unsigned long long* list, unsigned int* hist_q, int* maxbin_q) {
  s.valid = valid && thr_init < INFINITY;
  s.thr = s.valid ? thr_init : INFINITY;
  s.inv_q = s.valid ? inv_q : 0.f;
  s.qn = s.valid ? 1.0f / inv_q : 0.f;
  s.tb = (s.valid && thr_init > -INFINITY) ? score_bin(thr_init * inv_q) : -1;
  s.mb_cache = -1;
  s.nohist = false;
  s.cnt = 0;
  s.list = list;
  s.hist_q = hist_q;
  s.maxbin_q = maxbin_q;
}

// Raise thr from the global histogram (source 3).  Per-thread, no warp collectives.
// Bins are fetched 16 at a time (four independent 16-byte L2 loads in flight) rather than as a dependent chain
// of single loads.  The walk is out of line (it is long and rare) and takes / returns SCALARS: handing it the
// FilterState by reference would force the whole struct into local memory and cost the hot loop a local store
// per tile.
// Returns 0 if no bin edge with >= k' rows at or above it exists above bin `tb`; else (bin << 32) | raw-threshold bits.
static __device__ __noinline__ unsigned long long histogram_walk(const unsigned int* hist_q, int mb, int tb, float qn,
                                                                  int kprime) {
  const uint4* h4 = reinterpret_cast<const uint4*>(hist_q);
  const int g_lo = (tb + 1) >> 2;   // lowest group that may hold a bin > tb
  unsigned cum = 0;
  for (int g_hi = mb >> 2; g_hi >= g_lo; g_hi -= 4) {
    uint4 w[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) w[u] = (g_hi - u >= g_lo) ? __ldcg(h4 + g_hi - u) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int g = g_hi - u;
      const unsigned c[4] = {w[u].x, w[u].y, w[u].z, w[u].w};
#pragma unroll
      for (int j = 3; j >= 0; --j) {
        const int b = g * 4 + j;
        if (g >= g_lo && b <= mb && b > tb) {
          cum += c[j];
          if (cum >= static_cast<unsigned>(kprime))
            return (static_cast<unsigned long long>(b + 1) << 32) | __float_as_uint(bin_edge_raw(b, qn));
        }
      }
    }
  }
  return 0ull;
}
__device__ __forceinline__ bool filter_refresh(FilterState& s, int kprime) {
  if (!s.valid) return false;
  const int mb = __ldcg(s.maxbin_q);
  if (mb <= s.tb) return false;
  const unsigned long long r = histogram_walk(s.hist_q, mb, s.tb, s.qn, kprime);
  if (r == 0ull) return false;
  s.tb = static_cast<int>(r >> 32) - 1;
  s.thr = fmaxf(s.thr, __uint_as_float(static_cast<uint32_t>(r)));
  return true;
}

// When to refresh: every tile while the threshold is still moving fast, then ever more rarely
// (a stale threshold only costs a few extra appends).
__device__ __forceinline__ bool refresh_due(int it) {
  return it != 0 && (it < 8 || (it < 64 && (it & 7) == 0) || (it & 31) == 0);
}
// Shared-threshold variant (run_epilogue): walking the histogram costs a thread ~3 us, during which its
// accumulator stage is not drained.  The R units that scan different corpus ranges for the same queries
// would all compute the same number, so they take turns: at step `it` only unit it % R walks the histogram
// and publishes the result in gthr[q]; everybody else picks it up with one (prefetched) load per tile.
// The duty being spread over R units, it can come round far more often than a private refresh could.
__device__ __forceinline__ bool publish_due(int it) {
  return it != 0 && (it < 16 || (it < 64 && (it & 1) == 0) || (it & 7) == 0);
}
__device__ __forceinline__ void publish_threshold(FilterState& s, unsigned int* gthr_q, int kprime) {
  if (!s.valid) return;
  // thr may have been adopted from gthr since this thread last walked the histogram: skip the bins below it
  s.tb = max(s.tb, score_bin(s.thr * s.inv_q) - 1);
  filter_refresh(s, kprime);
  if (s.thr > -INFINITY) atomicMax(gthr_q, f32_ordered(s.thr));
}
__device__ __forceinline__ void adopt_threshold(FilterState& s, unsigned int ordered) {
  s.thr = fmaxf(s.thr, f32_from_ordered(ordered));   // 0 (nothing published) decodes to NaN, which fmaxf drops
}

// 1/||c|| of a chunk's rows: from shared memory (staged per tile) or, kGlobal, straight from the corpus-norm
// array through L1 (every lane reads the same address: one broadcast transaction).
template <bool kGlobal>
__device__ __forceinline__ float4 norm4(const float4* p) {
  if constexpr (kGlobal) return __ldg(p);
  else return *p;
}
template <bool kGlobal>
__device__ __forceinline__ float norm1(const float* p) {
  if constexpr (kGlobal) return __ldg(p);
  else return *p;
}

// Count one row of raw score t in the query's global histogram.  Every row must be counted AT MOST once:
// the counts are lower bounds on "rows of the corpus with a score in this bin", which is what makes a
// threshold read off the histogram safe.
__device__ __forceinline__ void hist_add(FilterState& s, float t) {
  const int b = score_bin(t * s.inv_q);
  atomicAdd(s.hist_q + b, 1u);
  if (b > s.mb_cache) {
    atomicMax(s.maxbin_q, b);
    s.mb_cache = b;
  }
}

__device__ __forceinline__ void filter_append(FilterState& s, float t, uint32_t row) {
  s.list[s.cnt] = pack_key(t, row);
  ++s.cnt;
  if (s.nohist) return;
  hist_add(s, t);
}

// Seeding pass over a unit's FIRST tile.  With no threshold yet, the plain filter appends (and counts) every
// row it sees until the histogram holds k' rows: a few hundred appends per thread (scattered 8-byte stores plus
// thousands of atomics per query landing on the same few histogram lines from every SM at once), a fixed cost
// of every search.  Instead the first tile is
// read twice: this pass only counts the two best group maxima of every 32-column chunk (two distinct rows,
// 16 per unit and tile, which is where the query's best rows so far are with overwhelming probability), all
// units' seeds then give the threshold, and the regular pass over the same accumulators appends the handful
// of rows above it - without counting them again.
// acc1 >= acc2: with whole_tile the two best rows seen so far in this thread's part of the tile (counted by the
// caller after the last chunk: 2 atomics per thread instead of 2 per chunk - enough when many units feed the
// same histogram, and an order of magnitude fewer same-line atomics in the first microseconds of a scan).
template <bool kGlobal = false>
__device__ __forceinline__ void seed_chunk(FilterState& s, const uint32_t (&v)[32], const float* invc32,
                                           bool whole_tile, float& acc1, float& acc2) {
  const float4* ic4 = reinterpret_cast<const float4*>(invc32);
  float m1 = -INFINITY, m2 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 w = norm4<kGlobal>(ic4 + j);
    const float a0 = __uint_as_float(v[4 * j + 0]) * w.x;
    const float a1 = __uint_as_float(v[4 * j + 1]) * w.y;
    const float a2 = __uint_as_float(v[4 * j + 2]) * w.z;
    const float a3 = __uint_as_float(v[4 * j + 3]) * w.w;
    const float x = fmaxf(fmaxf(fmaxf(a0, a1), fmaxf(a2, a3)), -INFINITY);   // a group of dead rows: NaN -> -inf
    m2 = fmaxf(m2, fminf(m1, x));
    m1 = fmaxf(m1, x);
  }
  if (whole_tile) {   // merge (m1 >= m2) into (acc1 >= acc2): the two largest of the four, distinct rows
    const float lo = fmaxf(fminf(acc1, m1), fmaxf(acc2, m2));
    acc1 = fmaxf(acc1, m1);
    acc2 = lo;
    return;
  }
  if (m1 > s.thr) hist_add(s, m1);
  if (m2 > s.thr) hist_add(s, m2);
}

// 32 accumulator columns of this thread's query; invc32 = the 32 matching 1/||c||.
template <bool kGlobal = false>
__device__ __forceinline__ void filter_chunk(FilterState& s, const uint32_t (&v)[32], const float* invc32,
                                             uint32_t row_base) {
  const float4* ic4 = reinterpret_cast<const float4*>(invc32);
  float g[8];   // maxima of the 8 groups of 4 columns (intermediates of the chunk maximum, kept for the slow path)
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 w = norm4<kGlobal>(ic4 + j);
    const float a0 = __uint_as_float(v[4 * j + 0]) * w.x;
    const float a1 = __uint_as_float(v[4 * j + 1]) * w.y;
    const float a2 = __uint_as_float(v[4 * j + 2]) * w.z;
    const float a3 = __uint_as_float(v[4 * j + 3]) * w.w;
    g[j] = fmaxf(fmaxf(a0, a1), fmaxf(a2, a3));   // fmaxf drops NaN (dead / out-of-range rows)
    m = fmaxf(m, g[j]);
  }
  if (m > s.thr) {
    // Rare per LANE but not per WARP while thresholds are still converging (1024 (query,row) pairs per warp
    // and chunk): walk only the groups of 4 that hold a survivor, so one lucky lane costs the warp a few
    // dozen instructions instead of 32 predicated append blocks.
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (g[j] > s.thr) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float t = __uint_as_float(v[4 * j + e]) * norm1<kGlobal>(invc32 + 4 * j + e);
          if (t > s.thr) filter_append(s, t, row_base + 4 * j + e);
        }
      }
    }
  }
}

__device__ __forceinline__ unsigned long long umax64(unsigned long long a, unsigned long long b) {
  return a > b ? a : b;
}
__device__ __forceinline__ unsigned long long umin64(unsigned long long a, unsigned long long b) {
  return a < b ? a : b;
}

// Warp-cooperative compaction of one list: bitonic sort of up to 256 keys (8 per lane,
// element i = j*32 + lane), keep the best k', return the k'-th score (source 2).
// Returns (bits of the k'-th score, or of -inf when the list is shorter) << 32 | entries kept - by value, so the
// caller's filter state stays in registers.
static __device__ __noinline__ unsigned long long warp_compact(unsigned long long* list, int cnt, int kprime, int lane) {
  constexpr uint32_t kFullMask = 0xFFFFFFFFu;
  unsigned long long k[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int idx = j * 32 + lane;
    k[j] = idx < cnt ? __ldcg(list + idx) : 0ull;
  }
#pragma unroll
  for (int k2 = 2; k2 <= 256; k2 <<= 1) {
#pragma unroll
    for (int st = k2 >> 1; st > 0; st >>= 1) {
      if (st >= 32) {
        const int js = st >> 5;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if ((j & js) == 0) {
            const int i = j * 32 + lane;
            const bool desc = (i & k2) == 0;
            const unsigned long long a = k[j], b = k[j | js];
            const unsigned long long hi = umax64(a, b), lo = umin64(a, b);
            k[j] = desc ? hi : lo;
            k[j | js] = desc ? lo : hi;
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int i = j * 32 + lane;
          const unsigned long long other = __shfl_xor_sync(kFullMask, k[j], st);
          const bool lower = (lane & st) == 0;
          const bool desc = (i & k2) == 0;
          k[j] = (lower == desc) ? umax64(k[j], other) : umin64(k[j], other);
        }
      }
    }
  }
  const int keep = cnt < kprime ? cnt : kprime;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int idx = j * 32 + lane;
    if (idx < keep) list[idx] = k[j];
  }
  const int e = kprime - 1;
  unsigned long long sel = 0ull;
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (j == (e >> 5)) sel = k[j];
  const unsigned long long kth = __shfl_sync(kFullMask, sel, e & 31);
  const float new_thr = cnt >= kprime ? key_score(kth) : -INFINITY;
  __syncwarp();
  return (static_cast<unsigned long long>(__float_as_uint(new_thr)) << 32) | static_cast<unsigned>(keep);
}

// Warp-collective: compact every lane's list that could overflow on the next chunk.
// `room`: appends that may happen before the next call (32 per chunk processed in between).
__device__ __forceinline__ void filter_compact_if_needed(FilterState& s, int kprime, int lane, int room = 32) {
  constexpr uint32_t kFullMask = 0xFFFFFFFFu;
  __syncwarp();
  unsigned need = __ballot_sync(kFullMask, s.cnt > kListCap - room);
  while (need) {
    const int src = __ffs(need) - 1;
    need &= need - 1;
    unsigned long long* l = reinterpret_cast<unsigned long long*>(
        __shfl_sync(kFullMask, reinterpret_cast<unsigned long long>(s.list), src));
    const int c = __shfl_sync(kFullMask, s.cnt, src);
    const unsigned long long r = warp_compact(l, c, kprime, lane);
    if (lane == src) {
      s.thr = fmaxf(s.thr, __uint_as_float(static_cast<uint32_t>(r >> 32)));
      s.cnt = static_cast<int>(static_cast<uint32_t>(r));
    }
  }
}


// Floats per row of the CTA's score buffer: 4 more than a tile row so that the 8 threads of a quarter warp, which
// read 16 bytes of 8 consecutive rows, hit 8 different groups of 4 banks.
constexpr int kScorePitch = kBlockN + 4;

// 32 consecutive scores of one row of the score buffer.
__device__ __forceinline__ void load_chunk(const float* src, uint32_t (&v)[32]) {
  const float4* s4 = reinterpret_cast<const float4*>(src);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 w = s4[j];
    v[4 * j + 0] = __float_as_uint(w.x);
    v[4 * j + 1] = __float_as_uint(w.y);
    v[4 * j + 2] = __float_as_uint(w.z);
    v[4 * j + 3] = __float_as_uint(w.w);
  }
}

// The whole epilogue role (thread <-> query) of the scan kernel: 128 threads (four warps), thread et filters the
// kBlockN scores of query row et of every tile of its unit [t0, t1).  scores: the CTA's score buffer (kBlockM rows of
// kScorePitch floats), filled by the wgmma warpgroups; sc_full / sc_empty hand it back and forth.  invc_stage: per-tile
// staging of the tile's 1/||c||, double-buffered by tile parity.
__device__ __forceinline__ void run_epilogue(const ScanParams& p, float (*invc_stage)[kBlockN],
                                             unsigned long long* sc_full, unsigned long long* sc_empty,
                                             const float* scores, int qb, int r, int t0, int t1, int et, int lane) {
  constexpr int kEpi = kBlockM;
  const int q = qb * kBlockM + et;
  const bool q_valid = q < p.B;
  const size_t list_id = static_cast<size_t>(qb * p.R + r) * kBlockM + et;
  FilterState fs;
  filter_init(fs, q_valid, q_valid ? p.thr_init[q] : INFINITY, q_valid ? p.inv_norm_q[q] : 0.f,
              p.cand + list_id * static_cast<size_t>(kListCap),
              p.hist + static_cast<size_t>(q_valid ? q : 0) * kHistBins, p.maxbin + (q_valid ? q : 0));
  const int n_iter = t1 - t0;
  // 1/||c|| of a tile's 256 rows are staged in shared memory behind one barrier of all epilogue threads per
  // tile (the warps wait there for the slowest of the previous tile); the NEXT tile's values travel in registers
  // while this one is processed, which hides their L2/HBM latency.
  float nx0 = 0.f, nx1 = 0.f;
  unsigned int* gthr_q = p.gthr + (q_valid ? q : 0);
  unsigned int ngt = 0u;   // published threshold, fetched one tile ahead
  if (n_iter > 0) {
    nx0 = __ldg(p.inv_norm_c + t0 * kBlockN + et);
    nx1 = __ldg(p.inv_norm_c + t0 * kBlockN + kEpi + et);
  }
  const float* srow = scores + et * kScorePitch;
  for (int it = 0; it < n_iter; ++it) {
    const int tile = t0 + it;
    const int row0 = tile * kBlockN;
    float* invc = invc_stage[it & 1];
    invc[et] = nx0;
    invc[kEpi + et] = nx1;
    if (it + 1 < n_iter) {
      nx0 = __ldg(p.inv_norm_c + (tile + 1) * kBlockN + et);
      nx1 = __ldg(p.inv_norm_c + (tile + 1) * kBlockN + kEpi + et);
    }
    adopt_threshold(fs, ngt);
    ngt = __ldcg(gthr_q);
    named_bar_sync(1, kEpi);
    if (publish_due(it) && r == it % p.R) publish_threshold(fs, gthr_q, p.kprime);   // overlaps this tile's wgmma
    mbar_wait(smem_u32(sc_full), static_cast<uint32_t>(it & 1));
    auto process = [&](uint32_t (&v)[32], int chunk) {
      filter_chunk(fs, v, invc + chunk * 32, static_cast<uint32_t>(row0 + chunk * 32));
      if (p.dbg_scores != nullptr && q_valid) {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int row = row0 + chunk * 32 + j;
          if (row < p.n_rows)
            p.dbg_scores[static_cast<size_t>(q) * p.n_rows + row] = __uint_as_float(v[j]) * invc[chunk * 32 + j];
        }
      }
    };
    uint32_t va[32], vb[32];
    if (it == 0) {
      // seeding pass (see seed_chunk): count the best rows of this tile, then take the threshold they give
      float sa1 = -INFINITY, sa2 = -INFINITY;
#pragma unroll 1
      for (int chunk = 0; chunk < kBlockN / 32; ++chunk) {
        load_chunk(srow + chunk * 32, va);
        seed_chunk(fs, va, invc + chunk * 32, false, sa1, sa2);
      }
      // the other units' seeds land within a microsecond or so of ours: a few short retries when the
      // histogram cannot hold k' rows yet but soon will
      const int tries = (p.R * 16 >= 2 * p.kprime) ? 6 : 1;
      for (int t = 0; t < tries; ++t) {
        const bool found = filter_refresh(fs, p.kprime);
        if (__all_sync(0xFFFFFFFFu, found || !fs.valid)) break;
        if (t + 1 < tries) __nanosleep(400);
      }
      if (fs.valid && fs.thr > -INFINITY) atomicMax(gthr_q, f32_ordered(fs.thr));
      fs.nohist = true;
    }
#pragma unroll 1
    for (int c2 = 0; c2 < kBlockN / 64; ++c2) {
      load_chunk(srow + (2 * c2) * 32, va);
      load_chunk(srow + (2 * c2 + 1) * 32, vb);
      process(va, 2 * c2);
      process(vb, 2 * c2 + 1);
      filter_compact_if_needed(fs, p.kprime, lane, 64);
      // seeding found nothing (too few units, or their seeds were late): keep looking while the tile is filtered
      if (it == 0 && fs.valid && fs.thr == -INFINITY) adopt_threshold(fs, __ldcg(gthr_q));
    }
    fs.nohist = false;
    mbar_arrive(smem_u32(sc_empty));
  }
  p.cand_cnt[list_id] = fs.cnt;
}

// Bounded-lag lockstep of the QB producers that stream the same corpus range: nobody runs
// more than kMaxLeadTiles ahead of the slowest, so a tile pulled from HBM by the first
// reader is still in L2 for the others (keeps DRAM traffic close to 1x the corpus).
__device__ __forceinline__ void lockstep_pace(volatile int* prog, int QB, int qb, int it, int max_lead) {
  if (QB <= 1 || (it & 1) != 0) return;   // every other tile: checking every tile costs ~10 % on short kernels
  prog[qb] = it;
  for (int o = 0; o < QB; ++o) {
    if (o == qb) continue;
    const long long w0 = clock64();
    while (prog[o] < it - max_lead) {
      __nanosleep(200);
      if (clock64() - w0 > (1ll << 24)) break;   // a pacing hint, never a correctness wait
    }
  }
}

}  // namespace rbk
