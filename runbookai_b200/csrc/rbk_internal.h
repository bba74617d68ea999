// rbk_internal.h — declarations shared by the kernels and the C-ABI translation unit.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace rbk {

// ---- tiling of the fused scan (rbk_scan.cu) ----
constexpr int kBlockM = 128;      // queries per CTA (two wgmma warpgroups of M = 64)
constexpr int kBlockN = 256;      // corpus rows per tile (wgmma N)
constexpr int kBlockK = 64;       // bf16 elements per pipeline stage (one 128-byte swizzle row)
constexpr int kStages = 4;        // smem ring depth
constexpr int kStageRows = 8;     // score rows a wgmma warpgroup hands to the epilogue per round
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

// The two passes of the large-k search (k_fetch up to RBK_MAX_K_FETCH_LARGE) run the same scan with another epilogue:
// count every row above a running threshold into the histogram, or emit every row above a fixed threshold.  Their
// extra fields live in a derived struct so that the top-k' kernel's parameter block stays as it is.
// kprime is k_fetch; in emit mode thr_init holds theta_q; cand / cand_cnt / dbg_scores are unused.
struct LargeScanParams : ScanParams {
  const double* q_eps;       // count: [B] error bound of the approximate cosine
  const long long* emit_off; // emit: [B] start of query q's segment of emit_rows
  const int* emit_cap;       // emit: [B] segment length C_q
  int* emit_cnt;             // emit: [B] rows emitted (zeroed per launch; exceeds emit_cap only through a bug)
  int* emit_rows;            // emit: flat local-row buffer
};
enum LargeScanMode { kScanCount = 1, kScanEmit = 2 };
cudaError_t launch_scan_large(const CUtensorMap& tmap_q, const CUtensorMap& tmap_c, const LargeScanParams& p,
                              LargeScanMode mode, cudaStream_t stream);
// The same kernels with fp16 operands (rbk_scan_f16.cu), for indexes created with RBK_INDEX_SCAN_F16: both tensor maps
// are then CU_TENSOR_MAP_DATA_TYPE_FLOAT16 maps of per-row scaled fp16 rows.
cudaError_t launch_scan_f16(const CUtensorMap& tmap_q, const CUtensorMap& tmap_c, const ScanParams& p,
                            cudaStream_t stream);
cudaError_t launch_scan_large_f16(const CUtensorMap& tmap_q, const CUtensorMap& tmap_c, const LargeScanParams& p,
                                  LargeScanMode mode, cudaStream_t stream);

// ---- ingest (rbk_ingest.cu) ----
// The exact-source rows of an index that keeps them (RBK_INDEX_KEEP_F64 / RBK_INDEX_KEEP_F32 /
// RBK_INDEX_KEEP_F32_SPLIT) are [cap][d] elements of x_elem bytes: 8 = float64, 4 = float32, 2 = the low halves of
// float32 values whose high halves are the scan copy `rows` (pitch dpad).  Every kernel that reads them widens each
// element to float64 on load and then runs the same operations in the same order, so a float32 row of float32-exact
// values gives the same bits as the float64 row.
//
// The split rule (x_elem 2), for a float32 with bits u: the scan copy is s = (u + 0x8000) >> 16 - bf16 rounded to
// nearest, ties away from zero, on the magnitude - and the low half is r = u & 0xFFFF.  Then u = ((s - (r >> 15)) << 16)
// | r exactly: r >= 0x8000 is exactly when the rounding carried into s.  Round-to-nearest-even cannot be undone so (a tie
// r == 0x8000 gives one s for two u).  A NaN's scan copy is the canonical bf16 NaN 0x7FFF, which still joins to a NaN.
struct F32Lo {
  uint16_t bits;
};
__host__ __device__ __forceinline__ uint16_t split_hi(uint32_t u) {
  return (u & 0x7FFFFFFFu) > 0x7F800000u ? static_cast<uint16_t>(0x7FFFu) : static_cast<uint16_t>((u + 0x8000u) >> 16);
}
__host__ __device__ __forceinline__ uint32_t split_join(uint32_t s, uint32_t r) { return ((s - (r >> 15)) << 16) | r; }
template <typename XT>
constexpr bool kIsSplit = std::is_same<XT, F32Lo>::value;
#ifdef __CUDACC__
__device__ __forceinline__ double split_f64(uint16_t s, uint16_t r) {
  return static_cast<double>(__uint_as_float(split_join(s, r)));
}
#endif
// src element type: 0 = f64, 1 = f32, 2 = bf16 bits.  src is device memory, row pitch = d.
// dst_x (nullable): exact-source rows (x_elem bytes per element, pitch d); a float32 destination takes only sources
// whose values are float32-exact (launch_find_not_f32 checks that first).
// slot_map (nullable, bulk overwrite): dst_rows / dst_x are the index's row 0 and source row r lands in row
// slot_map[r]; rows whose slot is tombstoned (dead_bits) are skipped and counted in *n_dead.
// f16: store the rows by the RBK_INDEX_SCAN_F16 rule (rbk_f16.cuh) instead of as bf16.  dst_x null with f16 only
// when src is the index's own exact rows (a tier change re-deriving the scan copy).
cudaError_t launch_convert_rows(const void* src, int src_type, int64_t n_rows, int d, int dpad,
                                uint16_t* dst_rows, void* dst_x, int x_elem, cudaStream_t stream,
                                const int64_t* slot_map = nullptr, const unsigned int* dead_bits = nullptr,
                                int* n_dead = nullptr, bool f16 = false);
// Norms of rows [first_row, first_row + n_items) of the index (or, with slot_map, of rows slot_map[i]; tombstoned
// ones skipped).  All array arguments are the index's BASE pointers.  rows_x_base (nullable, x_elem bytes per
// element): when given, norm2 comes from it and the bf16-vs-exact angle bound is max-ed into *eps_c_max (float bits
// in an int).
// f16: the rows are RBK_INDEX_SCAN_F16 fp16 rows (rows_x_base required); the angle is that of their rounding.
// dead_bits without slot_map (rows_x_base required; a tier change re-deriving every stored row): every row's norm2
// and angle are computed, but a tombstoned row's inv_norm stays NaN.
cudaError_t launch_row_norms(const uint16_t* rows_base, const void* rows_x_base, int x_elem, int64_t first_row,
                             int64_t n_items, int d, int dpad, float* inv_norm_base, double* norm2_base,
                             int* eps_c_max, cudaStream_t stream, const int64_t* slot_map = nullptr,
                             const unsigned int* dead_bits = nullptr, bool f16 = false);
cudaError_t launch_tombstone(const int64_t* dev_slots, int64_t n, int64_t n_rows, float* inv_norm,
                             unsigned int* dead_bits, int* n_killed, cudaStream_t stream);
// (rbk_gather.cu) Query b = the stored values of local row sel[b] (device [B], each < n_rows) as float64, into dst [B][d]: the exact
// row widened (x_elem 8 / 4), the split's float32 rebuilt from both halves (x_elem 2), or the bf16 scan copy widened
// (x_elem 0; never an RBK_INDEX_SCAN_F16 index, which keeps exact rows).  rows_x may be mapped host memory.  Adds the
// number of tombstoned rows among them to *n_dead, and gives each of those the query of zeros, which matches nothing.
cudaError_t launch_gather_rows(const uint16_t* rows, const void* rows_x, int x_elem, const unsigned int* dead_bits,
                               const int64_t* sel, int B, int d, int dpad, double* dst, int* n_dead,
                               cudaStream_t stream);
// (rbk_mmr.cu) The greedy MMR selection (rbk_index_search_mmr_f64), one block per query b: its candidates are rows
// [off[b], off[b + 1]) of x ([.][d] float64, device), at most max_m of them, with global slots slot[] and relevances
// rel[] at the same positions; k[b] picks at lambda_mult[b] go to row b of out_slots / out_scores ([B][K]), then
// -1 / quiet NaN.  Needs mmr_smem_bytes(max_m) of dynamic shared memory per block.
size_t mmr_smem_bytes(int max_m);
cudaError_t launch_mmr_select(const double* x, int d, const int64_t* off, const int64_t* slot, const double* rel,
                              const int* k, const double* lambda_mult, int B, int max_m, int K, int64_t* out_slots,
                              double* out_scores, cudaStream_t stream);
// *found = 1 if any of the n doubles at src (device or mapped host memory) is one a float32 cannot hold (else *found is
// left as it is): x is accepted iff it is NaN or (double)(float)x == x (so +-0, +-inf and float32 subnormals are, 0.1
// and 1e-300 are not).
cudaError_t launch_find_not_f32(const double* src, int64_t n, int* found, cudaStream_t stream);
// dst[i] = src[i] for n elements, from src_elem to dst_elem bytes (8 <-> 4; a float64 -> float32 copy only of values
// launch_find_not_f32 accepted): a tier change that widens or narrows the exact rows.  src_elem 2 (out of the split):
// n = n_rows * d elements, each joined with its high half in rows (pitch dpad).  A change INTO the split writes both
// halves with launch_convert_rows (x_elem 2) instead.
cudaError_t launch_convert_exact(const void* src, int src_elem, void* dst, int dst_elem, int64_t n,
                                 cudaStream_t stream, const uint16_t* rows = nullptr, int d = 0, int dpad = 0);

// ---- compaction (rbk_compact.cu) ----
// old_to_new [n_rows] (new local slot, -1 = tombstoned) from dead_bits by a two-level exclusive scan over the 32-row
// words.  Scratch: word_pref [ceil(n_rows / 32)], block_sum [ceil(n_rows / 32768)].  chunk_pref [n_chunks + 1]:
// [c] = live rows before row c * chunk_rows (a multiple of 32), [n_chunks] = all live rows.
cudaError_t launch_compact_map(const unsigned int* dead_bits, int64_t n_rows, int64_t chunk_rows, int* word_pref,
                               int* block_sum, long long* old_to_new, int* chunk_pref, cudaStream_t stream);
// Packs the live rows among source rows [s0, s0 + n) into staging row old_to_new[s] - d0: bf16 row (pitch dpad),
// exact row (x_elem bytes per element, pitch d; skipped when rows_x is null), norm2, inv_norm.
cudaError_t launch_compact_gather(const uint16_t* rows, const void* rows_x, int x_elem, const double* norm2,
                                  const float* inv_norm, const long long* old_to_new, int64_t s0, int64_t n,
                                  long long d0, int d, int dpad, uint16_t* st_rows, void* st_x, double* st_norm2,
                                  float* st_inv, int sm_count, cudaStream_t stream);

// ---- query preparation + finalize + exhaustive fallback + shard merge (rbk_finalize.cu) ----
struct QueryBuffers {
  uint16_t* q_bf16;    // [B][dpad] the scan's copy: bf16, or scaled fp16 for an RBK_INDEX_SCAN_F16 index
  double* q_f64;       // [B][d]
  double* q_norm2;     // [B] exact sequential sum of squares of the f64 query (reference's normA)
  float* q_inv_norm;   // [B] 1/||bf16(q)||, or 1/||h|| of the scaled fp16 copy (it carries the scale 2^-e)
  double* q_eps;       // [B] bound on |approx - exact| cosine for this query
  float* thr_init;     // [B]
};
// src_type: 0 = f64, 1 = f32 (device pointers, row pitch d)
// eps_c (nullable): device float, bound on the corpus-side quantisation angle (f64 sidecar indexes).
// with_norm2: also run the sequential normA chain (only the exact-scores path, which has no finalize kernel; a
// search leaves it to finalize).  scratch (nullable): hist | maxbin | gthr | progress of the first sub-batch (Bs
// queries, n_progress pacing slots), zeroed by the kernel.
// f16: the scan's copy follows the RBK_INDEX_SCAN_F16 rule (rbk_f16.cuh) and q_eps holds the angle of that rounding;
// a query is live (finite q_inv_norm) exactly when it would be for a bf16 index.
// min_each (nullable): each query's own min_score [B], in place of min_score.
cudaError_t launch_prep_queries(const void* src, int src_type, int B, int d, int dpad, double min_score,
                                const float* eps_c, const QueryBuffers& qb, cudaStream_t stream, bool with_norm2,
                                unsigned int* scratch, int Bs, int n_progress, bool f16 = false,
                                const double* min_each = nullptr);

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
  // the inverse of global(): the local row of global slot s, or -1 when this shard does not deal it
  __host__ __device__ int64_t local(int64_t s) const {
    if (block == 0) return s >= base ? s - base : -1;
    if (s < 0 || (s / block) % G != g) return -1;
    return (s / block / G) * block + s % block;
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
  const void* rows_x;       // nullable: exact-source rows (pitch d, x_elem of the launch); the re-rank reads them
  const double* row_norm2;
  int64_t n_rows;
  SlotLayout slot;
  QueryBuffers q;  // pointers already offset to the sub-batch
  long long* out_slots;   // [B][k_fetch]
  double* out_scores;     // [B][k_fetch]
  int* out_counts;        // [B]
  int* flags;             // [B] 1 = not provably exact -> exhaustive fallback
  // rbk_index_search_each_f64: each query's own cut and threshold, [B] offset to the sub-batch like q (nullable: k_fetch
  // and min_score for every query).  Then k_fetch is the row stride of the outputs, the largest k_each.
  const int* k_each;
  const double* min_each;
};
// rows_on_host: rows_x is mapped host memory (RBK_INDEX_ROWS_ON_HOST); the re-rank stages it with wide loads, more
// of them in flight, to cover the PCIe round trip.  Same scores either way.  x_elem: bytes per exact-row element (8, 4
// or 2; ignored when rows_x is null), here and in every launcher below that takes it.
cudaError_t launch_finalize(const FinalizeParams& p, bool rows_on_host, int x_elem, cudaStream_t stream);

struct ExactParams {
  const int* fail_list;  // [n_fail] query indices
  int n_fail;
  int d, dpad, k_fetch;
  double min_score;
  const uint16_t* rows;
  const void* rows_x;       // nullable: exact-source rows
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
  const int* k_each;         // nullable: per-query cut and threshold, indexed like q_f64 (k_fetch is then the stride)
  const double* min_each;
};
cudaError_t launch_exact_fallback(const ExactParams& p, int x_elem, cudaStream_t stream);

// ---- large-k search (rbk_finalize.cu): select between the two scan passes, exact re-rank after them ----
// theta [B] (raw domain) and cap [B] (C_q) from the count pass's histograms hist [B][kHistBins].
// A query whose q_eps is not below kEpsNone gets theta = +inf (the emit scan skips it) and C_q = n_rows; then
// launch_large_emit_all writes every live row into its segment.
// k_each (nullable): each query's own k_fetch [B], in place of k_fetch.
cudaError_t launch_large_select(const unsigned int* hist, const float* thr_init, const float* inv_norm_q,
                                const double* q_eps, int B, int k_fetch, int n_rows, float* theta, int* cap,
                                cudaStream_t stream, const int* k_each = nullptr);
cudaError_t launch_large_emit_all(const double* q_eps, const unsigned int* dead_bits, int64_t n_rows, int B,
                                  const long long* emit_off, int* emit_cnt, int* emit_rows, cudaStream_t stream);
struct LargeRerankParams {
  int B, d, dpad, k_fetch;
  double min_score;
  const uint16_t* rows;
  const void* rows_x;       // nullable: exact-source rows
  const double* row_norm2;
  SlotLayout slot;
  const double* q_f64;      // offset to the sub-batch, like every per-query array below
  const double* q_norm2;
  const long long* emit_off;
  const int* emit_cap;
  const int* emit_cnt;
  int* emit_rows;           // written only by the segmented sort's in-place tile sort
  double* cand_scores;      // parallel to emit_rows
  long long* out_slots;     // [B][k_fetch]
  double* out_scores;       // [B][k_fetch]
  int* out_counts;          // [B]
  int* overflow;            // += queries whose emit pass found more rows than C_q (a broken count)
  const int* k_each;        // nullable: per-query cut and threshold, offset to the sub-batch (k_fetch is then the
  const double* min_each;   // row stride, the largest k_each)
};

// The cut of k_fetch > RBK_MAX_K_FETCH_LARGE: a segmented sort in global memory.  Each query's segment of emit_rows /
// cand_scores is cut into tiles of kSortTile candidates (never two queries in one tile); every tile is sorted in
// shared memory, then adjacent sorted runs of the same query are merged pairwise, one pass per doubling, every run
// truncated to k_fetch entries.  The two buffers ping-pong: [0] is emit_rows / cand_scores themselves (each tile is
// sorted in place), [1] is the scratch below.
constexpr int kSortTile = 4096;
struct SegSortScratch {
  const int* tile_off;   // [B] first run-length slot of query q (tiles of the queries before it, in this group)
  double* scores;        // buffer [1], parallel to emit_rows
  int* rows;
  int* len[2];           // per-run passing lengths, one slot per tile (a run's length sits at its first tile)
  int max_tiles;         // most tiles of one query in this launch (sizes the grids and the number of passes)
};
// The exact fp64 re-score of every emitted candidate, then the cut to p.k_fetch entries per query, filled with
// -1 / NaN past the count: in shared memory, one block per query (sort null, p.k_fetch <= RBK_MAX_K_FETCH_LARGE), or
// the segmented sort above.  max_cap: largest emit_cap of the launch (sizes the scoring grid).  rows_on_host: as for
// launch_finalize; the scoring kernel then stages its candidates' rows in shared memory with coalesced loads.
// *launches: kernels enqueued.
cudaError_t launch_large_rerank(const LargeRerankParams& p, const SegSortScratch* sort, int max_cap,
                                bool rows_on_host, int x_elem, cudaStream_t stream, int* launches);

// rbk_index_similar_pairs_f64: B <= kMaxSubBatch queries that are the stored rows of global slots a0 + q, against the
// rows from local row r0 on.  The LargeRerankParams row pointers (rows, rows_x, row_norm2) then start at row r0, and
// so do the emitted rows; p.slot still maps local rows.  The re-score, then the drop of every candidate whose global slot
// is not above its query's (and, as in the sort, of scores below min_score and NaN), the segmented sort with no cut,
// counts [B] (each query's pairs), offsets [B] (their exclusive scan) and the pairs packed query after query into
// out_b / out_scores from offsets[q] on.  p.k_fetch and p.k_each are ignored.
struct PairsParams {
  int64_t a0, r0;
  int* counts;
  long long* offsets;
  long long* out_b;
  double* out_scores;
};
cudaError_t launch_pairs_rerank(const LargeRerankParams& p, const SegSortScratch& sort, int max_cap, bool rows_on_host,
                                int x_elem, const PairsParams& pp, cudaStream_t stream, int* launches);

// Exact fp64 cosine of every row for B prepared queries: out [B][n_rows], NaN = tombstoned / zero row.
cudaError_t launch_exact_scores(const uint16_t* rows, const void* rows_x, int x_elem, const double* row_norm2,
                                const unsigned int* dead_bits, int64_t n_rows, int d, int dpad, const double* q_f64,
                                const double* q_norm2, int B, double* out, cudaStream_t stream);

// slots/scores/counts/flags point at shard 0's arrays; shard g's arrays start g * <stride> bytes later.
// flags (nullable): per-shard exactness flags i32[B]; out_flags: i32[B+1] ([b] = OR over shards, [B] += dirty queries).
// k_each (nullable, device i32[B]): query b is cut at k_each[b]; k_fetch stays the row stride of every list.
cudaError_t launch_merge_shards(int G, int B, int k_fetch, const void* slots, const void* scores, const void* counts,
                                const void* flags, size_t slots_stride, size_t scores_stride, size_t counts_stride,
                                size_t flags_stride, long long* out_slots, double* out_scores, int* out_counts,
                                int* out_flags, cudaStream_t stream, const int* k_each = nullptr);

// Bound on the fp32 tensor-core accumulation + scaling error of an approximate cosine.
inline double accumulation_eps(int d) { return (double)(d + 8) * (1.0 / 4194304.0); }  // (d+8) * 2^-22

// The scan band (DESIGN.md §6): the scan's bound holds for a query or row whose largest finite element m has
// 2^-40 <= m < 2^40.  Then its bf16 copy is live, every product of two such copies' elements is below 2^81 (no fp32
// overflow for any d < 2^46), the elements that underflow in fp32 products change an approximate cosine by at most
// d 2^-126 / 2^-80 = d 2^-46 (far inside accumulation_eps), and normA / normB cannot underflow or overflow in float64.
// Outside it, a query the reference scores, or any such row in the index, gets a bound of kEpsNone or more: the
// first pass never proves it and the large-k search re-scores every live row.
constexpr double kScanBandLo = 9.094947017729282e-13;   // 2^-40
constexpr double kScanBandHi = 1099511627776.0;         // 2^40
__host__ __device__ inline bool in_scan_band(double m) { return m >= kScanBandLo && m < kScanBandHi; }
// A bound this wide (the whole range of a cosine) proves nothing; 3.2 is what an off-band row folds in.
constexpr double kEpsNone = 2.0;
constexpr float kEpsOffBand = 3.2f;

}  // namespace rbk
