// rbk_internal.h — declarations shared by the kernels and the C-ABI translation unit.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rbk {

// ---- tiling of the fused scan (rbk_scan.cu) ----
constexpr int kBlockM = 128;      // queries per CTA (two wgmma warpgroups of M = 64)
constexpr int kBlockN = 256;      // corpus rows per tile (wgmma N)
constexpr int kBlockK = 32;       // bf16 elements per pipeline stage (one 64-byte swizzle row)
constexpr int kStages = 3;        // smem ring depth
constexpr int kListCap = 256;     // entries per (CTA, query) candidate list
constexpr int kMaxKPrime = 128;   // candidates kept per query (k_fetch + margin)
constexpr int kScanThreads = 384; // warpgroup 0 epilogue, warpgroups 1-2 wgmma (+ TMA issue)
constexpr int kMaxSubBatch = 1024;  // queries per scan launch (8 query blocks)
constexpr int kMaxLeadTiles = 4;    // lockstep: max tiles a CTA may lead the slowest peer of its range
constexpr int kHistBins = 1024;     // per-query score histogram, cosine in [-1,1] -> bin width 1/512

struct ScanParams {
  const float* inv_norm_c;  // [rows padded to kBlockN], NaN = dead / out of range
  const float* thr_init;    // [B] initial threshold, raw domain (acc * inv_norm_c); -inf = none
  const float* inv_norm_q;  // [B] 1/||bf16(q)||
  unsigned int* hist;       // [B][kHistBins] scores of all appended rows (zeroed per launch)
  int* maxbin;              // [B] highest occupied histogram bin (zeroed per launch)
  unsigned int* gthr;       // [B] best published threshold per query, f32_ordered (0 = none; zeroed per launch)
  int* progress;            // [R][QB] tiles issued by each CTA's producer (zeroed per launch)
  unsigned long long* cand; // [QB][R][kBlockM][kListCap] packed keys
  int* cand_cnt;            // [QB][R][kBlockM]
  float* dbg_scores;        // nullable: [B][n_rows] raw-domain scores (validation aid)
  int n_rows;
  int B;        // queries in this launch
  int kprime;
  int dpad;     // padded row length (elements, a multiple of kBlockK)
  int max_lead_tiles;  // lockstep: tiles a producer may lead the slowest peer of its range
  int QB;       // query blocks
  int R;        // corpus ranges (CTAs that scan different tiles for the same queries) per query block
  int n_tiles;  // ceil(n_rows / kBlockN)
};

cudaError_t launch_scan(const CUtensorMap& tmap_q, const CUtensorMap& tmap_c, const ScanParams& p,
                        cudaStream_t stream);

// ---- ingest (rbk_ingest.cu) ----
// src element type: 0 = f64, 1 = f32, 2 = bf16 bits.  src is device memory, row pitch = d.
// dst_f64 (nullable): exact-source sidecar rows, pitch d.
// slot_map (nullable, bulk overwrite): dst_rows / dst_f64 are the index's row 0 and source row r lands in row
// slot_map[r]; rows whose slot is tombstoned (dead_bits) are skipped and counted in *n_dead.
cudaError_t launch_convert_rows(const void* src, int src_type, int64_t n_rows, int d, int dpad,
                                uint16_t* dst_rows, double* dst_f64, cudaStream_t stream,
                                const int64_t* slot_map = nullptr, const unsigned int* dead_bits = nullptr,
                                int* n_dead = nullptr);
// Norms of rows [first_row, first_row + n_items) of the index (or, with slot_map, of rows slot_map[i]; tombstoned
// ones skipped).  All array arguments are the index's BASE pointers.  rows_f64_base (nullable): when given,
// norm2 comes from it and the bf16-vs-f64 angle bound is max-ed into *eps_c_max (float bits in an int).
cudaError_t launch_row_norms(const uint16_t* rows_base, const double* rows_f64_base, int64_t first_row,
                             int64_t n_items, int d, int dpad, float* inv_norm_base, double* norm2_base,
                             int* eps_c_max, cudaStream_t stream, const int64_t* slot_map = nullptr,
                             const unsigned int* dead_bits = nullptr);
cudaError_t launch_tombstone(const int64_t* dev_slots, int64_t n, int64_t n_rows, float* inv_norm,
                             unsigned int* dead_bits, int* n_killed, cudaStream_t stream);

// ---- query preparation + finalize + exhaustive fallback + shard merge (rbk_finalize.cu) ----
struct QueryBuffers {
  uint16_t* q_bf16;    // [B][dpad]
  double* q_f64;       // [B][d]
  double* q_norm2;     // [B] exact sequential sum of squares of the f64 query (reference's normA)
  float* q_inv_norm;   // [B] 1/||bf16(q)||  (approximate-score scaling)
  double* q_eps;       // [B] bound on |approx - exact| cosine for this query
  float* thr_init;     // [B]
};
// src_type: 0 = f64, 1 = f32 (device pointers, row pitch d)
// eps_c (nullable): device float, bound on the corpus-side quantisation angle (f64 sidecar indexes).
// with_norm2: also run the sequential normA chain (only the exact-scores path, which has no finalize kernel; a
// search leaves it to finalize).  scratch (nullable): hist | maxbin | gthr | progress of the first sub-batch (Bs
// queries, n_progress pacing slots), zeroed by the kernel.
cudaError_t launch_prep_queries(const void* src, int src_type, int B, int d, int dpad, double min_score,
                                const float* eps_c, const QueryBuffers& qb, cudaStream_t stream, bool with_norm2,
                                unsigned int* scratch, int Bs, int n_progress);

// local row -> global slot.  Contiguous shards: slot_base + row.  A group that deals rows out block-cyclically over
// G devices (rbk_group.cu): device g's local row r is global slot ((r / block) * G + g) * block + r % block - still
// monotonic in r, so per-shard lists stay sorted by global slot among equal scores.
struct SlotLayout {
  int64_t base = 0;
  int32_t block = 0, G = 1, g = 0;   // block == 0: contiguous
  __host__ __device__ int64_t global(int64_t row) const {
    if (block == 0) return base + row;
    return ((row / block) * G + g) * block + row % block;
  }
};

struct FinalizeParams {
  const unsigned long long* cand;
  const int* cand_cnt;
  int QB, R, kprime, k_fetch, B, d, dpad;
  int block_m;  // queries per list block (kBlockM)
  int key_cap;  // keys staged in smem per query (set by launch_finalize)
  int q0;  // global index of the first query of this launch (sub-batch offset)
  double min_score;
  const uint16_t* rows;
  const double* rows_f64;   // nullable: exact-source sidecar (pitch d); the re-rank reads it instead of `rows`
  const double* row_norm2;
  int64_t n_rows;
  SlotLayout slot;
  QueryBuffers q;  // pointers already offset to the sub-batch
  long long* out_slots;   // [B][k_fetch]
  double* out_scores;     // [B][k_fetch]
  int* out_counts;        // [B]
  int* flags;             // [B] 1 = not provably exact -> exhaustive fallback
};
cudaError_t launch_finalize(const FinalizeParams& p, cudaStream_t stream);

struct ExactParams {
  const int* fail_list;  // [n_fail] query indices
  int n_fail;
  int d, dpad, k_fetch;
  double min_score;
  const uint16_t* rows;
  const double* rows_f64;   // nullable: exact-source sidecar
  const double* row_norm2;
  const unsigned int* dead_bits;  // tombstones
  int64_t n_rows;
  SlotLayout slot;
  const double* q_f64;
  const double* q_norm2;
  double* part_scores;   // [n_fail][n_blocks][k_fetch]
  int* part_rows;        // [n_fail][n_blocks][k_fetch]
  int* part_cnt;         // [n_fail][n_blocks]
  int n_blocks;
  long long* out_slots;
  double* out_scores;
  int* out_counts;
};
cudaError_t launch_exact_fallback(const ExactParams& p, cudaStream_t stream);

// Exact fp64 cosine of every row for B prepared queries: out [B][n_rows], NaN = tombstoned / zero row.
cudaError_t launch_exact_scores(const uint16_t* rows, const double* rows_f64, const double* row_norm2,
                                const unsigned int* dead_bits, int64_t n_rows, int d, int dpad, const double* q_f64,
                                const double* q_norm2, int B, double* out, cudaStream_t stream);

// slots/scores/counts/flags point at shard 0's arrays; shard g's arrays start g * <stride> bytes later.
// flags (nullable): per-shard exactness flags i32[B]; out_flags: i32[B+1] ([b] = OR over shards, [B] += dirty queries).
cudaError_t launch_merge_shards(int G, int B, int k_fetch, const void* slots, const void* scores, const void* counts,
                                const void* flags, size_t slots_stride, size_t scores_stride, size_t counts_stride,
                                size_t flags_stride, long long* out_slots, double* out_scores, int* out_counts,
                                int* out_flags, cudaStream_t stream);

// Bound on the fp32 tensor-core accumulation + scaling error of an approximate cosine.
inline double accumulation_eps(int d) { return (double)(d + 8) * (1.0 / 4194304.0); }  // (d+8) * 2^-22

}  // namespace rbk
