/*
 * rbk_knn.h — C ABI of the H100-native kNN engine behind RunbookAI's VectorStore.
 *
 * The reference has no FFI for this path; the seam is the TypeScript class
 * `VectorStore` (src/knowledge/store/vector-store.ts:24-333), whose hot loop is
 *     for (const [id, embedding] of this.embeddings)            (:210-215)
 *         score = cosineSimilarity(queryEmbedding, embedding)   (embedder.ts:168-184)
 *         if (score >= minScore) scored.push({id, score})
 *     scored.sort((a,b) => b.score - a.score)                   (:218)
 *     scored.slice(0, topK * 2)                                 (:221)
 * Each entry point below names the reference lines it replaces.  A Node N-API addon
 * (napi/rbk_napi.cc) or any other FFI binds exactly these symbols; INTEGRATION.md shows
 * the binding.  Plain C types only: no C++/torch/CUDA types cross this boundary
 * (CUDA streams and device pointers travel as void*).
 *
 * Conventions
 *   - "slot" = dense insertion index of a row = the reference's Map insertion position
 *     (SURVEY.md §8c S6/S9b).  The host side keeps the slot <-> "vec_<chunkId>" table.
 *   - Every function returns rbk_status; on failure rbk_last_error() holds the message
 *     the binding turns into `new Error(msg)`.  Nothing throws or aborts.
 *   - Inputs are borrowed for the duration of the call; outputs are caller-allocated.
 *   - An index is bound to ONE GPU.  A corpus sharded over several GPUs is either a
 *     group - rbk_group_*: one process, one handle, NCCL all-gather inside the search call - or one
 *     index per GPU in one process per GPU plus rbk_merge_topk_packed_device() after the
 *     caller's own exchange of the per-shard blocks.
 *   - Thread safety: calls on the same index are serialised by an internal mutex;
 *     different indexes are independent.
 *   - There is NO CPU fallback: without a CUDA device rbk_index_create fails with
 *     RBK_ECUDA.
 */
#ifndef RBK_KNN_H
#define RBK_KNN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RBK_ABI_VERSION 2
/* Largest k_fetch a single search accepts (the scan keeps k_fetch + margin <= 128). */
#define RBK_MAX_K_FETCH 112
/* Largest k_fetch of the large-k search (rbk_index_search_large_f64): 4 * limit for the reference's largest
 * limit (1000, knowledge-context.ts:150). */
#define RBK_MAX_K_FETCH_LARGE 4096
/* Widest row an index or group accepts: 1 <= dim <= RBK_MAX_DIM, else RBK_EINVAL. */
#define RBK_MAX_DIM (1 << 20)

typedef struct rbk_index rbk_index;

typedef enum {
  RBK_OK = 0,
  RBK_EINVAL = 1, /* bad argument */
  RBK_ENOMEM = 2, /* host or device allocation failed */
  RBK_ECUDA = 3,  /* CUDA runtime/driver error, or no device */
  RBK_ENCCL = 4,  /* NCCL missing or failing (rbk_group_* with more than one GPU) */
  RBK_EDIM = 5,   /* "Vectors must have the same length" (embedder.ts:169-171) */
  RBK_ENOTF32 = 6 /* a value is not exactly a float32 (only RBK_INDEX_KEEP_F32 and RBK_INDEX_KEEP_F32_SPLIT indexes and groups return it) */
} rbk_status;

int rbk_abi_version(void);
/* Message of the last failure on this thread (valid until the next failing call). */
const char* rbk_last_error(void);

/* ---- lifetime: `new VectorStore(dbPath)` / `close()` (vector-store.ts:28-32, :330) ---- */
/* dim: embedding length, 1 <= dim <= RBK_MAX_DIM (RBK_EINVAL outside, checked before the device).  device: CUDA
 * ordinal.  capacity_hint: rows to pre-allocate (0 = default; at least 1024 rows are mapped at creation, about 2*dim
 * bytes each, 10*dim with RBK_INDEX_KEEP_F64: 2 GiB and 10 GiB at RBK_MAX_DIM); the index grows on demand.  The device storage sits on virtual address ranges reserved
 * here for the most rows the device's memory could hold (min(2^31 - 512, total memory / device bytes per row)); a
 * capacity_hint above that fails with RBK_ENOMEM.  Growth maps more physical memory behind the same addresses: nothing
 * is copied, so growing to capacity C needs C's storage, not the old and the new at once.  The capacity doubles
 * (whole 256-row tiles); if the doubled capacity cannot be backed, it grows to exactly the rows needed instead, and
 * only if that fails too does the call return RBK_ENOMEM, with the index unchanged.  A device without CUDA virtual
 * memory management fails with RBK_ECUDA. */
rbk_status rbk_index_create(int32_t dim, int32_t device, int64_t capacity_hint, rbk_index** out);
/* flags: RBK_INDEX_KEEP_F64 keeps, next to the bf16 rows the scan reads, the ORIGINAL values of every appended
 * row as float64 (8*dim bytes per row; f32/bf16 inputs are widened exactly).  The exact re-rank then uses them:
 * results are the reference's fp64 cosine bit for bit for ARBITRARY float64 embeddings (the SQLite BLOBs of
 * vector-store.ts:71-88), not only for bf16-representable ones.  The scan's error bound grows by the largest
 * angle between a row and its bf16 rounding, so more queries may take the exhaustive path on near-tied data.
 * The scan's bound covers only rows and queries whose largest finite element m has 2^-40 <= m < 2^40 (the scan band,
 * DESIGN.md §6).  A query the reference scores (finite, not all zero) outside the band skips the scan and is answered
 * by the exhaustive kernel.  Once ANY such row has been stored (in any tier; it stays so until rbk_index_clear), every
 * top-k search of the index takes the exhaustive kernel and every large-k search re-scores every live row: exact, at
 * the cost of the whole corpus per query. */
#define RBK_INDEX_KEEP_F64 1u
/* RBK_INDEX_F64_ON_HOST (only together with RBK_INDEX_KEEP_F64 or RBK_INDEX_KEEP_F32, else RBK_EINVAL; also spelled
 * RBK_INDEX_ROWS_ON_HOST): the [capacity][dim] exact rows (float64 below; float32 at half the bytes with KEEP_F32)
 * live in pinned, mapped host memory (cudaHostAlloc Mapped | Portable) instead of on the GPU; every other buffer stays
 * where it is.  Answers are bit-identical to a KEEP_F64 index on the device fed the same calls - slots, scores, counts,
 * exactness flags, fallback and retry decisions, compaction maps: the same values go through the same operations in
 * the same order, only the bytes come over PCIe.  Device memory per row at d = 1536 drops from 15,372 to 3,084 bytes
 * (about 5x the rows per GPU); host RAM pays 8*dim bytes per row (12 KB at d = 1536), and growing the capacity holds
 * the old and the new buffer at once (peak old + new): the host rows are one cudaHostAlloc buffer, reallocated and
 * copied on growth and on rbk_index_trim, unlike the device buffers, which grow in place.  The scan is unchanged.  Cost: each search reads k'*8*dim
 * bytes of host rows per query (k' = candidates re-ranked, <= 128; about 590 KB at k_fetch 20, d = 1536), the large-k
 * search 8*dim bytes per emitted candidate, and the rare exhaustive fallback / rbk_index_exact_scores_f64 the whole
 * corpus, all at PCIe speed; appends write the rows over PCIe.  Every write to the host rows is stream-ordered (a kernel
 * or copy on the index stream, or the host after a synchronisation), so searches enqueued earlier never see a
 * half-written row.  The placement is fixed until rbk_index_set_tier. */
#define RBK_INDEX_F64_ON_HOST 2u
/* RBK_INDEX_KEEP_F32 (exclusive with RBK_INDEX_KEEP_F64: both return RBK_EINVAL): keeps the exact rows as float32,
 * [capacity][dim] at 4*dim bytes per row, instead of float64.  Only float32-exact values are stored: a double x is
 * accepted iff it is NaN or (double)(float)x == x (so +-0, +-inf and float32 subnormals are; 0.1, 1e-300 and 1e39 are
 * not).  rbk_index_append_f32 / _bf16 always qualify.  rbk_index_append_f64, rbk_index_append_f64_device,
 * rbk_index_overwrite_f64 and rbk_index_overwrite_f64_batch check every value of the call on the device before anything
 * is written (overwrite_f64_batch before its tombstoned-slot rule writes the live slots); a call holding any other value
 * returns RBK_ENOTF32 and leaves the index exactly as it was - size, count, rows, norms, the corpus-side error bound,
 * tombstone bits, and so the answers of every later search (a capacity grown during the call may stay grown).  NaN
 * elements may lose their payload bits.  A group refuses the whole call before any member writes.
 * The contract: a KEEP_F32 index fed the same calls answers exactly as a KEEP_F64 index with the same other flags -
 * slots, fp64 scores and counts, -1 / NaN tails, exactness flags, retry and fallback decisions and the stats counters,
 * debug scores, compaction maps, the corpus-side bound and the scan-band rule.  It holds because a float32 row widened to
 * double IS the float64 row: every kernel widens each element on load and runs the same operations in the same order.
 * What changes is the bytes: 9,228 instead of 15,372 device bytes per row at d = 1536 on the device tier (the row
 * ceiling below uses them), 6,144 instead of 12,288 pinned host bytes with RBK_INDEX_ROWS_ON_HOST, and half the bytes
 * read per row by the re-rank, the exhaustive fallback and rbk_index_exact_scores_f64. */
#define RBK_INDEX_KEEP_F32 64u
/* The placement flag under its general name: with either keep bit, the exact rows (float64 or float32) live in pinned,
 * mapped host memory, as described for RBK_INDEX_F64_ON_HOST (host RAM then pays 8*dim or 4*dim bytes per row). */
#define RBK_INDEX_ROWS_ON_HOST RBK_INDEX_F64_ON_HOST
/* RBK_INDEX_SCAN_F16 (only together with RBK_INDEX_KEEP_F64 or RBK_INDEX_KEEP_F32, else RBK_EINVAL; combines with
 * RBK_INDEX_F64_ON_HOST):
 * the scan reads fp16 rows instead of bf16, at the same 2 bytes per element.  Each row x (and each query) is stored
 * scaled by its own power of two, h_i = RNE_f16(x_i * 2^e) with e = 15 - E, E the frexp exponent of max |x_i| over the
 * finite elements (so max|x| * 2^e is in [2^14, 2^15)); results that would be subnormal are stored as signed zeros.
 * fp16 keeps 11 significant bits against bf16's 8, so the scan's error bound - whose rounding terms are the angles
 * between a row or query and its stored copy - is several times tighter (DESIGN.md §6): fewer batches need the wide
 * retry, and the large-k search emits fewer candidates.  Answers are those of a KEEP_F64 index without the flag: the
 * same slots and fp64 scores, bit for bit, including the scan-band rule above (decided on the float64 row or query,
 * not on the scaled copy).  The placement is fixed until rbk_index_set_tier; read the stored bits with
 * rbk_index_read_rows_f16. */
#define RBK_INDEX_SCAN_F16 16u
/* RBK_INDEX_KEEP_F32_SPLIT (a keep bit: exclusive with RBK_INDEX_KEEP_F64, RBK_INDEX_KEEP_F32 and RBK_INDEX_SCAN_F16, all
 * RBK_EINVAL; combines with RBK_INDEX_ROWS_ON_HOST): keeps float32 exact rows like RBK_INDEX_KEEP_F32, with the same
 * accepted values, the same checks and the same RBK_ENOTF32 contract, but stores each float32 only once.  Its high 16
 * bits live in the bf16 scan copy, which is rounded for that purpose, and only the low 16 bits are kept beside it: the
 * exact rows cost 2*dim bytes per row instead of 4*dim.  For a float32 with bits u the scan copy is (u + 0x8000) >> 16
 * (bf16 rounded to nearest with ties away from zero, on the magnitude; a NaN becomes the bf16 NaN 0x7FFF), the low half
 * is u & 0xFFFF, and u = ((s - (r >> 15)) << 16) | r rebuilds the value exactly (a NaN stays a NaN, its payload may be
 * lost).  With RBK_INDEX_ROWS_ON_HOST only the low halves move to pinned, mapped host memory (2*dim bytes per row); the
 * scan copy stays on the device.
 * The contract: fed the same calls, a split index gives the answers of a KEEP_F32 index with the same placement - slots,
 * fp64 scores, counts, -1 / NaN tails, compaction maps, RBK_ENOTF32 refusals with the index untouched, and the scan-band
 * rule.  Where no stored value has a low half of exactly 0x8000 (a tie, where ties-away and ties-to-even round apart) it
 * also has the same stored scan bits, corpus-side bound, debug scores, exactness flags, retry and fallback decisions and
 * stats counters; otherwise only those decision-side outputs may differ.  rbk_index_read_rows_bf16 returns the scan
 * copy.  At d = 1536: 6,156 device bytes per row on the device tier (9,228 with KEEP_F32), and 3,072 pinned host bytes
 * per row with RBK_INDEX_ROWS_ON_HOST (6,144 with KEEP_F32); the row ceiling and rbk_index_storage_bytes count them. */
#define RBK_INDEX_KEEP_F32_SPLIT 128u
rbk_status rbk_index_create_ex(int32_t dim, int32_t device, int64_t capacity_hint, uint32_t flags, rbk_index** out);
void rbk_index_destroy(rbk_index* idx); /* NULL is a no-op */
/* The index's creation flags as they are now (RBK_INDEX_KEEP_F64, RBK_INDEX_KEEP_F32 or RBK_INDEX_KEEP_F32_SPLIT |
 * RBK_INDEX_F64_ON_HOST | RBK_INDEX_SCAN_F16); 0 for NULL. */
uint32_t rbk_index_flags(const rbk_index* idx);
/* Change the storage tier of an index with exact rows in place, from the rows it holds: move them between the device
 * and pinned host memory (RBK_INDEX_F64_ON_HOST), switch the scan between bf16 and fp16 (RBK_INDEX_SCAN_F16), and keep
 * them as float64 or float32 (RBK_INDEX_KEEP_F64 / RBK_INDEX_KEEP_F32), in any combination, without reloading.
 *   - flags: a flag set rbk_index_create_ex accepts with one of the keep bits (an exact copy cannot be made from bf16
 *     rows, and dropping it would change the answers); anything else returns RBK_EINVAL with the index untouched.
 *   - Widening (KEEP_F32 -> KEEP_F64) always succeeds given the memory.  Narrowing (KEEP_F64 -> KEEP_F32) succeeds only if
 *     every stored slot [0, size()), live or tombstoned, holds float32-exact values (the rule of RBK_INDEX_KEEP_F32);
 *     otherwise it returns RBK_ENOTF32, checked before anything changes.  Either way the new exact-row buffer is
 *     allocated and filled before the old one is released: peak memory is the old plus the new exact rows.
 *     RBK_INDEX_KEEP_F32_SPLIT takes part in every such change, in and out, the same way (narrowing from KEEP_F64 is
 *     checked the same way); entering or leaving it also rewrites the scan copy under the target's rounding and
 *     recomputes the norms and the corpus-side bound, like a change of scan type.
 *   - The current flags are a no-op (RBK_OK).  The member indexes of a group refuse the call (RBK_EINVAL):
 *     rbk_group_set_tier changes them together.
 *   - Every answer stays bit for bit: slots, fp64 scores, counts, -1 / NaN tails, exactness flags, compaction maps; so
 *     do size(), count(), slot_base, the capacity and the stats counters.
 *   - Afterwards the index is what rbk_index_create_ex with `flags`, fed the same calls, would be: the same stored scan
 *     bits (tombstoned slots included; the one exception is a NaN element of a bf16 input, whose payload bits the bf16
 *     tier's direct copy kept and a re-derivation does not), inv_norm and norm2, rbk_index_storage_bytes, and the
 *     row ceiling that later growth can reach, min(2^31 - 512, total device memory / device bytes per row) of the new
 *     tier.  Moving the rows to the host maps the device buffers' existing physical memory at new, larger address
 *     ranges (nothing is copied, peak device memory does not grow).
 *   - The corpus-side error bound is recomputed under the new scan type as the largest angle over every stored slot,
 *     live or tombstoned (a change of placement alone keeps it).  It is never larger than that of an index created
 *     with `flags`; after overwrites or compaction it may be smaller, and then fewer batches may take the wide retry or
 *     the fallback.  Once an off-band row has been stored (see RBK_INDEX_KEEP_F64), the bound stays one that proves
 *     nothing until rbk_index_clear.
 *   - Every allocation - the pinned [capacity][dim] buffer, the device memory of the float64 rows, the new address
 *     ranges - happens before anything changes: RBK_ENOMEM (and RBK_EINVAL) leaves the index exactly as it was.
 *     Moving the rows to the device fails so when the capacity is above the device tier's row ceiling (rbk_index_trim
 *     first, or stay).  That guarantee covers the allocations only: a CUDA error while the rows move (RBK_ECUDA,
 *     which poisons the context anyway) may leave the index part-way changed; the allocations it no longer needs are
 *     released.
 *   - Synchronous.  Searches enqueued earlier (rbk_index_search_device_async) finish first, on the old tier, because the
 *     index's work is stream-ordered.  Cost: one pass of the float64 rows from one side of PCIe to the other (placement),
 *     and the ingest kernels over every stored row (scan type; they read the rows over PCIe when they are on the host). */
rbk_status rbk_index_set_tier(rbk_index* idx, uint32_t flags);

/* Run all device work of this index on the given cudaStream_t (NULL = the index's own
 * stream).  Lets a host framework time the engine with events on its current stream. */
rbk_status rbk_index_set_stream(rbk_index* idx, void* cuda_stream);
/* Global slot of local row 0 (row-sharded corpora; SURVEY.md §8e).  Default 0. */
rbk_status rbk_index_set_slot_base(rbk_index* idx, int64_t slot_base);

/* ---- mutation: loadEmbeddings / addChunk(s) / deleteDocument / clear
 *      (vector-store.ts:56-66, :93-183, :285-297, :322-325) ---- */
/* rows: n_rows x dim, row-major.  f64 is the SQLite BLOB layout (little-endian float64,
 * vector-store.ts:71-88).  Values are stored as bf16 (round-to-nearest-even); the index
 * is exact for inputs representable in bf16 (DESIGN.md §3).  first_slot_out (nullable)
 * receives the LOCAL slot of the first appended row.  `rows` (host memory, pageable or
 * page-locked, or device memory for the *_device variants) has been consumed when the
 * call returns; the conversion itself may still be running on the index's stream. */
rbk_status rbk_index_append_f64(rbk_index* idx, const double* rows, int64_t n_rows, int64_t* first_slot_out);
rbk_status rbk_index_append_f32(rbk_index* idx, const float* rows, int64_t n_rows, int64_t* first_slot_out);
rbk_status rbk_index_append_bf16(rbk_index* idx, const uint16_t* rows, int64_t n_rows, int64_t* first_slot_out);
/* Same, rows already in device memory on the index's GPU (bulk load without a PCIe hop).  The rows are read on the
 * index's stream, which is not ordered after any other stream: work that writes them on another stream (a framework's
 * current stream, say) must be complete, or that stream must be the index's (rbk_index_set_stream), before the call. */
rbk_status rbk_index_append_bf16_device(rbk_index* idx, const void* dev_rows, int64_t n_rows,
                                        int64_t* first_slot_out);
/* f64 rows (the BLOB layout) already on the device, e.g. a sidecar file read with GPUDirect or staged by the host
 * framework in large pinned chunks. */
rbk_status rbk_index_append_f64_device(rbk_index* idx, const void* dev_rows, int64_t n_rows, int64_t* first_slot_out);
/* `this.embeddings.set(id, e)` on an existing id keeps its Map position (S9b). */
rbk_status rbk_index_overwrite_f64(rbk_index* idx, int64_t local_slot, const double* row);
/* The same for n rows at once - a re-embedded document (addChunks over existing ids, vector-store.ts:135-183):
 * rows[i] (n x dim, f64) replaces local_slots[i].  One call, one host round trip for the whole batch.  A slot that
 * is tombstoned stays dead and makes the call return RBK_EINVAL after the LIVE slots of the batch have been
 * written (the host mirror never overwrites a deleted id, so this is a caller bug, not a data path).  A slot named
 * more than once takes its LAST row, as Map.set twice would. */
rbk_status rbk_index_overwrite_f64_batch(rbk_index* idx, const int64_t* local_slots, int64_t n, const double* rows);
/* `this.embeddings.delete(id)`: the rows stop matching.  Their slots stay allocated (size() does not shrink) until
 * rbk_index_compact reclaims them. */
rbk_status rbk_index_tombstone(rbk_index* idx, const int64_t* local_slots, int64_t n);
/* Reclaim the slots of tombstoned rows.  The live rows move down to local slots 0 .. count()-1 in their current
 * order (the Map's iteration order survives, so tie order and every search answer are unchanged up to the
 * renumbering); afterwards size() == count().  old_to_new (nullable) receives, for every local slot s < size()
 * before the call, its new local slot, or -1 if s was tombstoned; old_to_new_len must then be >= that size()
 * (RBK_EINVAL otherwise, index untouched).  Liveness is the tombstone bits alone: a zero row stays, in its place.
 * slot_base is kept, so global slots stay slot_base + local.  Capacity is kept: later appends reuse the reclaimed
 * slots.  Without tombstones nothing moves and the identity map is returned.  Staging is one 64 MB buffer, allocated
 * before the first row moves (RBK_ENOMEM leaves the index untouched).  Not available for the member indexes of a
 * group (RBK_EINVAL): rbk_group_compact compacts them together.  Synchronous.  Searches enqueued before the call (rbk_index_search_device_async) run first,
 * because the index's work is stream-ordered; their results carry the OLD slots. */
rbk_status rbk_index_compact(rbk_index* idx, int64_t* old_to_new, int64_t old_to_new_len);
rbk_status rbk_index_clear(rbk_index* idx);
/* Give memory back.  Synchronises the index's stream first, so searches enqueued earlier
 * (rbk_index_search_device_async) finish before anything they read goes away.  Then sets the capacity to that of a
 * new index holding size() rows, round_up(max(size(), 1024), 256), and unmaps the device storage beyond it (the pinned
 * host rows of RBK_INDEX_F64_ON_HOST are reallocated at that capacity); releases every search, compaction and staging
 * scratch buffer, device and pinned, which the next call that needs one re-grows; and drops the captured search graph
 * and the corpus tensor map.  Answers never change and nothing is renumbered (unlike rbk_index_compact, so the member
 * indexes of a group may be trimmed).  Trim after rbk_index_compact or rbk_index_clear to return their slots' bytes.
 * Storage is unmapped in whole physical chunks of at most 256 MiB: afterwards the mapped device bytes exceed
 * rbk_index_storage_bytes by less than one chunk per device buffer (five at most).  Growing again maps memory, it does
 * not copy. */
rbk_status rbk_index_trim(rbk_index* idx);
int64_t rbk_index_count(const rbk_index* idx); /* live rows  */
int64_t rbk_index_size(const rbk_index* idx);  /* slots used, tombstones included */
int32_t rbk_index_dim(const rbk_index* idx);
/* Persistent corpus storage at the current capacity, in bytes: bf16 rows, inv_norm, norm2, tombstone bits and the
 * exact rows (8*dim bytes per row with KEEP_F64, 4*dim with KEEP_F32), split by where they live.  Search and compaction scratch are not counted.  Either output
 * may be NULL. */
rbk_status rbk_index_storage_bytes(const rbk_index* idx, int64_t* device_bytes, int64_t* pinned_host_bytes);
/* Copy stored rows back (bf16 bits), for tests and for reload sidecars.  RBK_EINVAL on an RBK_INDEX_SCAN_F16 index. */
rbk_status rbk_index_read_rows_bf16(rbk_index* idx, int64_t first_local_slot, int64_t n_rows, uint16_t* out);
/* The same for an RBK_INDEX_SCAN_F16 index: the stored, scaled fp16 bits (RBK_EINVAL on any other index). */
rbk_status rbk_index_read_rows_f16(rbk_index* idx, int64_t first_local_slot, int64_t n_rows, uint16_t* out);

/* ---- search: the scan + sort + cut of VectorStore.search (vector-store.ts:207-221)
 *      and findMostSimilar (embedder.ts:189-202), batched over B queries ---- */
/*
 * queries: B x query_dim row-major, HOST memory.  query_dim != dim -> RBK_EDIM, message
 * "Vectors must have the same length".  For each query b the call returns the first
 * out_counts[b] <= k_fetch entries of: all live rows with cosine >= min_score (fp64,
 * inclusive; pass -INFINITY for "no threshold"), ordered by score descending, ties by
 * ascending slot.  Scores are the reference's fp64 cosine, bit for bit, for the stored
 * (bf16-exact) rows.  out_slots are GLOBAL (slot_base + local).  Unused tail entries of
 * row b are slot -1 / score NaN.  kernel_ms_out (nullable): device time of the call.
 */
rbk_status rbk_index_search_f64(rbk_index* idx, const double* queries, int32_t B, int32_t query_dim,
                                int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                int32_t* out_counts, float* kernel_ms_out);
rbk_status rbk_index_search_f32(rbk_index* idx, const float* queries, int32_t B, int32_t query_dim,
                                int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                int32_t* out_counts, float* kernel_ms_out);
/* Device-resident variant: queries (f32, B x dim) and all outputs are device pointers on
 * the index's GPU; work is enqueued on the index stream and the call returns after the
 * exactness check of the batch (it synchronises the stream once). */
rbk_status rbk_index_search_device(rbk_index* idx, const void* dev_queries_f32, int32_t B, int32_t k_fetch,
                                   double min_score, void* dev_out_slots_i64, void* dev_out_scores_f64,
                                   void* dev_out_counts_i32);

/* Up to RBK_MAX_K_FETCH_LARGE hits per query (callers of the reference pass limit: 1000, knowledge-context.ts:150,
 * which becomes k_fetch = 4000 through the hybrid retriever): exactly the contract of rbk_index_search_f64 - same
 * order, threshold, NaN / tombstone rules and bit-identical fp64 scores - for 1 <= k_fetch <= 4096.  k_fetch <= 112
 * is accepted too and gives the same answer as rbk_index_search_f64.  Two scans of the corpus (count, then emit the
 * rows the count proved may belong to the answer), an exact fp64 re-rank of those rows and the cut to k_fetch in
 * shared memory; one extra host round trip between the scans.  Host queries and outputs, synchronous; batches over
 * 1024 queries are split.  Device memory is bounded by a fixed per-pass budget (256 MiB of candidates and results, at
 * least one query per pass): the count scan runs once for the batch, then the queries go in contiguous groups that fit
 * the budget, each group costing one emit scan and one copy of its results to the host through a pinned buffer the
 * index keeps (rbk_index_trim releases it).  kernel_ms_out is the time of the whole call on the device's stream.
 * Fails with RBK_ECUDA, never with a wrong answer, if an emit scan finds more rows than the count scan bounded (a
 * bug). */
rbk_status rbk_index_search_large_f64(rbk_index* idx, const double* queries, int32_t B, int32_t query_dim,
                                      int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                      int32_t* out_counts, float* kernel_ms_out);

/* Any number of hits per query - the reference's VectorStore.search has no ceiling on topK (vector-store.ts:207-221):
 * exactly the contract of rbk_index_search_large_f64 (same order, threshold, NaN / tombstone rules, bit-identical
 * fp64 scores, -1 / NaN tail, RBK_EDIM / RBK_EINVAL on the same arguments) for any int32 k_fetch >= 1.
 * k_fetch <= RBK_MAX_K_FETCH_LARGE runs rbk_index_search_large_f64 itself.  Above it the same pipeline keeps
 * k_eff = min(k_fetch, rbk_index_count()) entries per query on the device (no query can have more hits) and, in
 * place of the cut in shared memory, sorts each query's candidates in global memory after the exact re-score; the
 * per-pass budget, the query groups and the pinned copy-back are the same, so device memory never grows with k_fetch.
 * Fails with RBK_ECUDA, never with a wrong answer, if an emit scan finds more rows than the count scan bounded (a
 * bug). */
rbk_status rbk_index_search_unbounded_f64(rbk_index* idx, const double* queries, int32_t B, int32_t query_dim,
                                          int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                          int32_t* out_counts, float* kernel_ms_out);

/* Each query of a batch at its own k_fetch[b] (>= 1) and min_score[b] (any value but NaN; -INFINITY = none), in one
 * call: row b of the result is exactly what rbk_index_search_unbounded_f64 returns for query b alone with B = 1 at
 * k_fetch[b] and min_score[b] - the same slots, the same fp64 score bits, the same count - and so, where those accept
 * the k, what rbk_index_search_large_f64 and rbk_index_search_f64 return.  The rows of out_slots / out_scores are
 * K = max_b k_fetch[b] entries long ([B][K]); entries [out_counts[b], K) are slot -1 / the quiet NaN
 * 0x7FF8000000000000.  Argument checks, before any device work and in the order of the other searches: a null array
 * with B > 0 or a k_fetch[b] < 1 is RBK_EINVAL, the wrong query_dim RBK_EDIM, a NaN min_score[b] RBK_EINVAL; B = 0 is
 * RBK_OK.  One call adds 1 to the searches counter and B to the queries counter.
 * The whole batch takes one route, picked by K: up to RBK_MAX_K_FETCH the fused top-k' scan at k' = k'(K), every query
 * cut, counted and proven at its own k and threshold (a query whose proof fails is re-answered, at its own parameters,
 * by the wide rescan and then the exhaustive kernel); above it the two-scan large-k pipeline for every query, each one
 * cut at its own k_eff (min(k_fetch[b], count()) when K > RBK_MAX_K_FETCH_LARGE, else k_fetch[b]).  So callers that want
 * different k and thresholds share one pass over the corpus (two for the large-k route), where one search per distinct
 * (k, min_score) would cost a pass each.  Host queries in, host results out; synchronous. */
rbk_status rbk_index_search_each_f64(rbk_index* idx, const double* queries, int32_t B, int32_t query_dim,
                                     const int32_t* k_fetch, const double* min_score, int64_t* out_slots,
                                     double* out_scores, int32_t* out_counts, float* kernel_ms_out);

/* The exact fp64 cosine of EVERY row, out_scores[b * size() + slot], NaN for tombstoned / zero rows (which the
 * reference's `>= minScore` drops too, S3), for a host that applies the threshold, the stable sort and the cut itself
 * (vector-store.ts:212-221).  One fp64 pass over the corpus per query and 8 * size() bytes per query to the host; a
 * search for more hits than RBK_MAX_K_FETCH_LARGE is far cheaper through rbk_index_search_unbounded_f64. */
rbk_status rbk_index_exact_scores_f64(rbk_index* idx, const double* queries, int32_t B, int32_t query_dim,
                                      double* out_scores);

/* Stored rows as queries ("the chunks most like this stored chunk"): row b of the result is exactly what
 * rbk_index_search_each_f64 returns for one host query - the stored values of global slot query_slots[b] - at
 * k_fetch[b] and min_score[b]: the same slots, fp64 score bits, count and -1 / quiet-NaN tail in the [B][K] layout,
 * K = max_b k_fetch[b].  The stored values are the float64 row (RBK_INDEX_KEEP_F64), the float32 row widened
 * (RBK_INDEX_KEEP_F32), the float32 joined from the scan copy's high half and the kept low half, widened
 * (RBK_INDEX_KEEP_F32_SPLIT), or the bf16 row widened (no exact rows), on either placement and scan type; a NaN element
 * may lose its payload bits.  The query's own slot is part of its answer.  Slots are global: an index answers only for
 * [slot_base, slot_base + size()).  Argument checks, before any device work and in the order of
 * rbk_index_search_each_f64: a null array with B > 0, a k_fetch[b] < 1, a NaN min_score[b] or a slot the index does
 * not hold is RBK_EINVAL.  A tombstoned slot is RBK_EINVAL too, found on the device by the gather and reported after the
 * round trip the search makes anyway; the outputs are then unspecified and nothing else changes.  B = 0 is RBK_OK.  One
 * call adds 1 to the searches counter and B to the queries counter.  The slots are answered in chunks of 1024 queries,
 * each taking the route of its own largest k, so device memory does not grow with B (a pass over every row of the
 * index needs one chunk's scratch).  Synchronous. */
rbk_status rbk_index_search_slots_f64(rbk_index* idx, const int64_t* query_slots, int32_t B, const int32_t* k_fetch,
                                      const double* min_score, int64_t* out_slots, double* out_scores,
                                      int32_t* out_counts, float* kernel_ms_out);

/* Every pair of stored rows at or above a cosine threshold ("which chunks are near-duplicates of each other"): each
 * pair of live global slots a < b with first_slot <= a < *next_slot whose fp64 cosine of the stored values (those
 * rbk_index_search_slots_f64 uses as a query) is >= min_score (inclusive; -INFINITY = every pair).  The score is bit for
 * bit the reference's cosineSimilarity(row_a, row_b), which is symmetric in the bits - every product commutes exactly
 * and sqrt(na) * sqrt(nb) == sqrt(nb) * sqrt(na) - so keeping only b > a loses nothing.  out_a[i], out_b[i],
 * out_scores[i] for i < *n_out, ascending a, then score descending, ties by ascending b: the entries with first element a
 * are exactly those of rbk_index_search_slots_f64({a}, count(), min_score) whose slot is > a, in the same order with
 * the same score bits.  A tombstoned a contributes nothing (it is not refused); zero rows and rows containing NaN pair
 * with nothing.
 * Paging: the call returns the pairs of the longest run of query rows from first_slot that fits in max_pairs entries
 * (never part of a row's pairs) and sets *next_slot to the first row not answered, slot_base + size() when the pass is
 * complete; the next call continues there, and the pages concatenate to one call with a large enough buffer.  The rows
 * go in chunks of 1024: when the buffer fills, the rest of that chunk's work is discarded and re-done by the next call.
 * Argument checks, before any device work and in the order of the other searches: a null output, a NaN min_score, a
 * first_slot outside [slot_base, slot_base + size()] or max_pairs < max(size(), 1) (so that every call makes progress)
 * is RBK_EINVAL, and so is a call on a group member.  first_slot == slot_base + size() is RBK_OK with no pairs.  One call
 * adds 1 to the searches counter and *next_slot - first_slot to the queries counter.
 * How: per chunk [a0, a0 + Q), the gather of rbk_index_search_slots_f64, then the large-k pipeline over the rows from a0
 * on only (the scans start at the tile holding a0), with theta_q from min_score and the query's error bound alone (no
 * k), the exact re-score, the drop of b <= a, the global-memory sort with no cut, and the pairs packed query after query;
 * one round trip brings back the counts, another the rows that fit.  Device memory stays within the large-k per-pass
 * budget however many pairs there are.  kernel_ms_out (nullable): device time of the call.  Synchronous. */
rbk_status rbk_index_similar_pairs_f64(rbk_index* idx, double min_score, int64_t first_slot, int64_t max_pairs,
                                       int64_t* out_a, int64_t* out_b, double* out_scores, int64_t* n_out,
                                       int64_t* next_slot, float* kernel_ms_out);

/* fetch_k[b] * dim must not exceed this: at most 256 MiB of float64 candidate rows staged per query. */
#define RBK_MMR_MAX_FETCH_ELEMS (1 << 25)
/* Diverse hits by maximal marginal relevance (MMR): k[b] of query b's fetch_k[b] best candidates, picked greedily so that
 * each pick is relevant to the query and unlike the picks before it.  lambda_mult[b] in [0, 1] weighs the two (1: the
 * plain ranking).  For query b the result is defined exactly as follows.
 *  1. Candidates: c_0 .. c_{m-1} with relevance r_0 .. r_{m-1} are exactly row b of rbk_index_search_each_f64 at
 *     k_fetch = fetch_k[b], min_score = min_score[b]: the same slots and fp64 score bits in the same order (score
 *     descending, ties by ascending slot).  Candidate index i is the rank in that list.
 *  2. Pair similarity: s(i, j) is the reference's cosineSimilarity of the stored values of the two rows - the values
 *     rbk_index_search_slots_f64 uses as a query: the float64 row, the float32 row widened, the split float32 rebuilt
 *     from its two halves, or the bf16 row widened.  Its bits are symmetric in i and j.
 *  3. Greedy: the first pick is c_0.  For each later pick, every unpicked i has red_i, the largest non-NaN s(i, j) over
 *     the picks j so far, or NaN if all of them are NaN (a new s replaces red_i only if it is strictly greater, or if
 *     red_i is NaN), and mmr_i = lambda * r_i - (1 - lambda) * red_i, one correctly rounded fp64 operation per step in
 *     this order: t = 1.0 - lambda, a = lambda * r_i, c = t * red_i, mmr = a - c.  The pick is the i that ranks first
 *     under a total order: a NaN mmr ranks below every number, then the larger value wins, then the smaller i.
 *  4. Output: out_counts[b] = min(k[b], m); row b of out_slots / out_scores ([B][K], K = max_b k[b]) holds the picks in
 *     selection order, each pick's global slot and its relevance r; the tail is slot -1 and the quiet NaN
 *     0x7FF8000000000000, as in rbk_index_search_each_f64.  No mmr value is returned.
 * Invariants: at lambda = 1 the result is the first min(k, m) entries of the search_each row whenever no s is +-inf;
 * k = 1 gives c_0; a group gives the answers of a single index holding the same rows.
 * Argument checks, before any device work and in the order of rbk_index_search_each_f64: a null array with B > 0, a
 * k[b] < 1, a fetch_k[b] < k[b], a fetch_k[b] > RBK_MAX_K_FETCH_LARGE or a fetch_k[b] * dim > RBK_MMR_MAX_FETCH_ELEMS is
 * RBK_EINVAL; then the wrong query_dim is RBK_EDIM; then a NaN min_score[b] or a lambda_mult[b] outside [0, 1] (NaN
 * included) is RBK_EINVAL.  B = 0 is RBK_OK.  One call adds 1 to the searches counter and B to the queries counter.
 * How: queries go in chunks of 1024.  Each chunk runs the search_each pipeline at its largest fetch_k, then the
 * candidates' rows are gathered as float64 into device scratch, for contiguous query groups whose rows fit the large-k
 * per-pass budget (256 MiB), and one block per query runs the greedy selection on the device (rbk_mmr.cu).  The lock is
 * held throughout, so the candidates and their rows come from the same state.  rbk_index_trim releases the scratch.
 * kernel_ms_out (nullable): device time of the whole call.  Synchronous. */
rbk_status rbk_index_search_mmr_f64(rbk_index* idx, const double* queries, int32_t B, int32_t query_dim,
                                    const int32_t* k, const int32_t* fetch_k, const double* lambda_mult,
                                    const double* min_score, int64_t* out_slots, double* out_scores,
                                    int32_t* out_counts, float* kernel_ms_out);

/* Enqueue-only variant: nothing is synchronised, the call returns as soon as the kernels are queued on the index
 * stream, so batches pipeline back to back and an exchange step (all-gather + rbk_merge_topk_packed_device) can be
 * queued behind it without a host round trip in between.  dev_out_flags_i32[B]: 0 = the answer of query b is
 * proven exact (the normal case), 1 = not proven (more near-ties around the k_fetch-th hit than the candidate
 * margin holds).  The caller checks the flags when it eventually synchronises - for a sharded corpus AFTER the
 * merge, whose out_flags OR the shards' flags - and re-answers a batch that has any dirty query with the
 * synchronous rbk_index_search_device (which rescans with a wide margin / falls back to the exhaustive kernel).
 * All four outputs may point into a packed block (below). */
rbk_status rbk_index_search_device_async(rbk_index* idx, const void* dev_queries_f32, int32_t B, int32_t k_fetch,
                                         double min_score, void* dev_out_slots_i64, void* dev_out_scores_f64,
                                         void* dev_out_counts_i32, void* dev_out_flags_i32);

/* Merge G per-shard result lists (layout [G][B][k_fetch], each sorted as above, device
 * memory, e.g. the output of an all-gather) into [B][k_fetch] by (score desc, slot asc).
 * Enqueued on cuda_stream; no synchronisation. */
rbk_status rbk_merge_topk_device(int32_t device, void* cuda_stream, int32_t G, int32_t B, int32_t k_fetch,
                                 const void* dev_slots_i64, const void* dev_scores_f64, const void* dev_counts_i32,
                                 void* dev_out_slots_i64, void* dev_out_scores_f64, void* dev_out_counts_i32);

/* Same merge for G PACKED per-shard blocks laid end to end (what ONE all-gather of each rank's block
 * produces).  Block layout, rbk_packed_block_bytes(B, k_fetch) bytes: slots i64[B*k_fetch] | scores
 * f64[B*k_fetch] | counts i32[B] (padded to 16 bytes) | flags i32[B] (padded to 16 bytes; starts at
 * rbk_packed_flags_offset).  rbk_index_search_device(_async) can write straight into a block: pass block,
 * block + B*k_fetch*8, block + B*k_fetch*16 (and block + rbk_packed_flags_offset for the flags).
 * dev_out_flags_i32 (nullable): i32[B+1]; [b] = OR of the shards' flags of query b, [B] += number of dirty
 * queries of this call (a running count the caller zeroes, so a pipelined loop checks once at the end). */
int64_t rbk_packed_block_bytes(int32_t B, int32_t k_fetch);
int64_t rbk_packed_flags_offset(int32_t B, int32_t k_fetch);
rbk_status rbk_merge_topk_packed_device(int32_t device, void* cuda_stream, int32_t G, int32_t B, int32_t k_fetch,
                                        const void* dev_blocks, void* dev_out_slots_i64, void* dev_out_scores_f64,
                                        void* dev_out_counts_i32, void* dev_out_flags_i32);

/* ---- one corpus over several GPUs behind ONE handle (SURVEY.md §8b/§8e; rbk_group.cu) ----
 * What a single host process (RunbookAI is one Node process) uses to shard `this.embeddings` over the GPUs of a
 * box: one index per device, rows dealt out block-cyclically (4096-row blocks, so the corpus may grow at sync
 * time), every search = H2D of the queries to every GPU, the fused scan on every GPU, ONE ncclAllGather of the packed
 * per-GPU blocks over NVLink, a merge kernel on device_ids[0], one D2H and ONE host synchronisation - all inside
 * rbk_group_search_*.  Slots are GLOBAL insertion indices, exactly as for a single index; results are identical
 * to a single index holding the same rows (ids and fp64 scores bit for bit, ties by ascending slot).
 * NCCL is looked up at run time (dlopen "libnccl.so.2"); a group of more than one GPU fails with RBK_ENCCL if it
 * is missing, a one-GPU group never touches it.  device_ids may name a device more than once (e.g. {0, 0, 0}: three
 * members on GPU 0, each with its own stream): such a group creates no NCCL communicator and gathers the members'
 * blocks to device_ids[0] with device copies instead; its answers are those of any other group.  Mutation and search
 * semantics, limits (k_fetch <= RBK_MAX_K_FETCH) and error conventions are those of the rbk_index_* call of the same
 * name. */
typedef struct rbk_group rbk_group;
rbk_status rbk_group_create(int32_t dim, const int32_t* device_ids, int32_t n_devices, int64_t capacity_hint,
                            uint32_t flags /* RBK_INDEX_KEEP_F64 or RBK_INDEX_KEEP_F32 [| RBK_INDEX_F64_ON_HOST]
                                              [| RBK_INDEX_SCAN_F16]: every member */,
                            rbk_group** out);
void rbk_group_destroy(rbk_group* grp); /* NULL is a no-op */
rbk_status rbk_group_append_f64(rbk_group* grp, const double* rows, int64_t n_rows, int64_t* first_slot_out);
rbk_status rbk_group_append_f32(rbk_group* grp, const float* rows, int64_t n_rows, int64_t* first_slot_out);
rbk_status rbk_group_append_bf16(rbk_group* grp, const uint16_t* rows, int64_t n_rows, int64_t* first_slot_out);
rbk_status rbk_group_overwrite_f64_batch(rbk_group* grp, const int64_t* slots, int64_t n, const double* rows);
rbk_status rbk_group_tombstone(rbk_group* grp, const int64_t* slots, int64_t n);
rbk_status rbk_group_clear(rbk_group* grp);
/* Reclaim the slots of tombstoned rows across the group: rbk_index_compact in GLOBAL slots.  The live rows move down
 * to global slots 0 .. rbk_group_count()-1 in their current global order, moving between devices where the
 * block-cyclic layout puts their new slot elsewhere; afterwards every member holds exactly the rows and per-row state
 * that a new group of the same devices and flags would hold after appending the survivors in order, size() ==
 * count(), and later appends land at count().  old_to_new (nullable) receives, for every global slot s <
 * rbk_group_size() before the call, its new global slot, or -1 if s was tombstoned; old_to_new_len must then be >=
 * that size (RBK_EINVAL otherwise, group untouched).  No slot or score changes except through the map.  Every
 * allocation (one staging buffer of 64 MB, or one 4096-row block if that is more, per member) happens before the first
 * row moves (RBK_ENOMEM leaves the group untouched); tombstone bits that disagree with a member's count() return
 * RBK_ECUDA before anything moves.  Every member's corpus-side error bound becomes the largest of them (answers are
 * unchanged; retry and fallback counts may differ from those of a new group).  Capacity is kept: follow with
 * rbk_group_trim to return it.  Without tombstones nothing moves and the identity map is returned.  Synchronous; uses
 * no NCCL.  The members themselves refuse rbk_index_compact (RBK_EINVAL). */
rbk_status rbk_group_compact(rbk_group* grp, int64_t* old_to_new, int64_t old_to_new_len);
/* rbk_index_trim on every member, and the group's own exchange buffers released. */
rbk_status rbk_group_trim(rbk_group* grp);
/* rbk_index_set_tier on every member together (read the flags of any member with rbk_index_flags): every member's
 * checks (RBK_ENOTF32 for a narrowing) and allocations happen before any member changes, so RBK_ENOMEM and RBK_ENOTF32
 * leave the whole group as it was.  Synchronous; uses no NCCL. */
rbk_status rbk_group_set_tier(rbk_group* grp, uint32_t flags);
int64_t rbk_group_count(const rbk_group* grp); /* live rows */
int64_t rbk_group_size(const rbk_group* grp);  /* slots used, tombstones included */
int32_t rbk_group_devices(const rbk_group* grp);
rbk_index* rbk_group_member(rbk_group* grp, int32_t i); /* the i-th device's index (stats, tests); owned by the group */
int64_t rbk_group_redone_batches(const rbk_group* grp); /* batches re-answered because a shard's proof failed */
rbk_status rbk_group_search_f32(rbk_group* grp, const float* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                                double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                                float* device_ms_out);
rbk_status rbk_group_search_f64(rbk_group* grp, const double* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                                double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                                float* device_ms_out);
/* rbk_index_search_large_f64 over the group: the count scan on every GPU and one wait for all of them, then per query
 * group - the members' candidates and result blocks taken together fit the same per-pass budget - the emit scan,
 * re-rank and cut on every GPU, the same all-gather and merge as rbk_group_search_f64, and the copy into the caller's
 * arrays.  A one-GPU group never touches NCCL. */
rbk_status rbk_group_search_large_f64(rbk_group* grp, const double* queries, int32_t B, int32_t query_dim,
                                      int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                      int32_t* out_counts, float* device_ms_out);
/* rbk_index_search_unbounded_f64 over the group (any k_fetch >= 1; up to RBK_MAX_K_FETCH_LARGE it is
 * rbk_group_search_large_f64): the pipeline of rbk_group_search_large_f64, with the sort in global memory as the cut
 * and k_eff = min(k_fetch, rbk_group_count()) entries per query on every GPU. */
rbk_status rbk_group_search_unbounded_f64(rbk_group* grp, const double* queries, int32_t B, int32_t query_dim,
                                          int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                          int32_t* out_counts, float* device_ms_out);
/* rbk_index_search_each_f64 over the group: every member takes the route of the batch's largest k, the merge cuts
 * query b at its own k_fetch[b] (k_eff on the large-k route), and a batch re-answered after a member's proof failed is
 * re-answered at the same per-query parameters.  Same arguments, checks, layout and answers as the index call. */
rbk_status rbk_group_search_each_f64(rbk_group* grp, const double* queries, int32_t B, int32_t query_dim,
                                     const int32_t* k_fetch, const double* min_score, int64_t* out_slots,
                                     double* out_scores, int32_t* out_counts, float* device_ms_out);
/* rbk_index_search_slots_f64 over the group: the member that holds each global slot gathers its stored values into the
 * group's pinned query staging (one round trip per chunk of 1024 queries, which also reports a tombstoned slot), then
 * rbk_group_search_each_f64 runs from there.  A slot the group does not hold (>= rbk_group_size()) is RBK_EINVAL.  Same
 * arguments, checks, layout and answers as the index call on a single index holding the same rows. */
rbk_status rbk_group_search_slots_f64(rbk_group* grp, const int64_t* query_slots, int32_t B, const int32_t* k_fetch,
                                      const double* min_score, int64_t* out_slots, double* out_scores,
                                      int32_t* out_counts, float* device_ms_out);
/* rbk_index_similar_pairs_f64 over the group's global slots [0, rbk_group_size()): the same arguments, checks, paging
 * and answers as a single index holding the same rows.  Per chunk the owners gather its rows into the group's pinned
 * query staging, every member pairs them with its own rows from the chunk's first slot on, and the host merges the
 * members' sorted lists per query.  Every member's counters take the call.  Uses no NCCL. */
rbk_status rbk_group_similar_pairs_f64(rbk_group* grp, double min_score, int64_t first_slot, int64_t max_pairs,
                                       int64_t* out_a, int64_t* out_b, double* out_scores, int64_t* n_out,
                                       int64_t* next_slot, float* device_ms_out);
/* rbk_index_search_mmr_f64 over the group: the candidates come from rbk_group_search_each_f64 (global slots); per query
 * group the members that hold them gather their rows into pinned staging, and the selection runs on device_ids[0].
 * Uses no NCCL beyond that of rbk_group_search_each_f64.  Same arguments, checks, layout and answers as the index call
 * on a single index holding the same rows; rbk_group_trim releases the staging. */
rbk_status rbk_group_search_mmr_f64(rbk_group* grp, const double* queries, int32_t B, int32_t query_dim,
                                    const int32_t* k, const int32_t* fetch_k, const double* lambda_mult,
                                    const double* min_score, int64_t* out_slots, double* out_scores,
                                    int32_t* out_counts, float* device_ms_out);

/* ---- introspection ---- */
typedef struct {
  int64_t searches;         /* search calls */
  int64_t queries;          /* queries answered */
  int64_t fallback_queries; /* queries re-answered by the exhaustive fp64 kernel (after the wide retry) */
  int64_t scan_launches;    /* launches of the fused scan kernel */
  int64_t kernel_launches;  /* all kernel launches made by this index */
  float last_scan_ms;       /* device time of the scan kernel(s) of the last synchronous search (async: of the last finished scan) */
  float last_total_ms;      /* device time of the whole last search */
  int32_t last_kprime;      /* candidates kept per query by the last scan */
  int32_t sm_count;
  int32_t last_ring_stages; /* smem ring depth of the last scan kernel */
  int32_t retry_batches;    /* batches scanned a second time with the widest candidate margin after a failed proof */
  double scan_ms_total;     /* device time of all scan kernels that have FINISHED so far (CUDA events around every launch) */
  int64_t scans_timed;      /* number of scan launches folded into scan_ms_total */
  int64_t graph_replays;    /* small-batch host searches served by replaying the captured CUDA graph (prep + scan + finalize + copies) */
} rbk_stats;
/* Never blocks: folds in the scans that have finished and returns. */
rbk_status rbk_index_stats(rbk_index* idx, rbk_stats* out);

/* Debug/validation aid (tests only): run the scan on `queries` (host f32, B x dim) and
 * return the approximate scores of every (query,row) pair, B x size() floats (host).
 * NaN marks tombstoned/zero rows. */
rbk_status rbk_index_debug_scores_f32(rbk_index* idx, const float* queries, int32_t B, float* out_scores);

#ifdef __cplusplus
}
#endif
#endif /* RBK_KNN_H */
