// rbk_index_impl.h — the index object behind the opaque `rbk_index*` of include/rbk_knn.h and the host-side
// helpers shared by the two translation units that implement the C ABI: rbk_capi.cu (one index = one GPU) and
// rbk_group.cu (one group = one index per GPU + the NCCL exchange, all behind one call).
#pragma once
#include <string.h>

#include <functional>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/rbk_knn.h"
#include "rbk_internal.h"

namespace rbk {
namespace impl {

rbk_status fail(rbk_status st, const std::string& msg);
rbk_status cuda_fail(cudaError_t e, const char* what);
#define CK(expr)                                                    \
  do {                                                              \
    cudaError_t _e = (expr);                                        \
    if (_e != cudaSuccess) return ::rbk::impl::cuda_fail(_e, #expr); \
  } while (0)

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  cudaError_t ensure(size_t want) {
    if (want <= n) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&p), want * sizeof(T));
    if (e == cudaSuccess) n = want;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
};
template <typename T>
struct PinBuf {
  T* p = nullptr;
  size_t n = 0;
  cudaError_t ensure(size_t want) {
    if (want <= n) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr;
    n = 0;
    cudaError_t e = cudaMallocHost(reinterpret_cast<void**>(&p), want * sizeof(T));
    if (e == cudaSuccess) n = want;
    return e;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    n = 0;
  }
};

// One device corpus buffer on a reserved virtual address range (CUDA virtual memory management).  Physical chunks
// are mapped from `base` on as the index grows and unmapped from the end by rbk_index_trim, so `base` does not move and
// a growth copies nothing.  The one exception is rbk_index_set_tier moving the f64 rows to the host: it maps the same
// chunks at a larger range (raising the row ceiling) and the base pointers move there.
struct VmRange {
  struct Chunk {
    CUmemGenericAllocationHandle handle;
    size_t bytes;
  };
  CUdeviceptr base = 0;
  size_t reserved = 0, mapped = 0;   // [base, base + mapped) is backed
  std::vector<Chunk> chunks;         // in address order from base
};

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// Entries [k_eff, k_fetch) of each of the B result rows of k_fetch entries: slot -1, score NaN (a large-k search
// keeps at most k_eff = count() hits per query).
inline void fill_result_tail(int64_t* slots, double* scores, int32_t B, int32_t k_fetch, int32_t k_eff) {
  if (k_eff >= k_fetch) return;
  const uint64_t nan_bits = 0x7FF8000000000000ull;   // the quiet NaN the device kernels write
  double nan;
  memcpy(&nan, &nan_bits, sizeof nan);
  for (int32_t b = 0; b < B; ++b) {
    const size_t o = static_cast<size_t>(b) * k_fetch;
    for (int32_t i = k_eff; i < k_fetch; ++i) {
      slots[o + i] = -1;
      scores[o + i] = nan;
    }
  }
}

// Byte layout of one search's results as one block, so that they and the exactness flags move in one copy:
//   slots i64 [B][k_fetch] | scores f64 [B][k_fetch] | counts i32 [B] | flags i32 [B]
// counts and flags each padded to 16 bytes.  The C ABI publishes it (rbk_packed_block_bytes / rbk_packed_flags_offset):
// a device group all-gathers these blocks, and so do multi_device.py and the addon.
struct ResultBlock {
  int64_t B, nk, off_scores, off_counts, off_flags, bytes;
  ResultBlock(int32_t B_, int32_t k_fetch)
      : B(B_), nk(B * k_fetch), off_scores(nk * 8), off_counts(nk * 16), off_flags(off_counts + (B * 4 + 15) / 16 * 16),
        bytes(off_flags + (B * 4 + 15) / 16 * 16) {}
  long long* slots(void* base) const { return static_cast<long long*>(base); }
  double* scores(void* base) const { return reinterpret_cast<double*>(static_cast<char*>(base) + off_scores); }
  int* counts(void* base) const { return reinterpret_cast<int*>(static_cast<char*>(base) + off_counts); }
  int* flags(void* base) const { return reinterpret_cast<int*>(static_cast<char*>(base) + off_flags); }
  // copies a host block out to the caller's arrays
  void unpack(const void* h, int64_t* out_slots, double* out_scores, int32_t* out_counts) const {
    const char* p = static_cast<const char*>(h);
    memcpy(out_slots, p, sizeof(int64_t) * nk);
    memcpy(out_scores, p + off_scores, sizeof(double) * nk);
    memcpy(out_counts, p + off_counts, sizeof(int32_t) * B);
  }
  // copies a host block of k entries per query out to the caller's rows of k_fetch >= k entries, out_* pointing at
  // the block's first query; entries [k, k_fetch) of each row get slot -1, score NaN
  void unpack_rows(const void* h, int32_t k_fetch, int64_t* out_slots, double* out_scores, int32_t* out_counts) const {
    const char* p = static_cast<const char*>(h);
    const int64_t k = B > 0 ? nk / B : 0;
    for (int64_t b = 0; b < B; ++b) {
      memcpy(out_slots + b * k_fetch, p + sizeof(int64_t) * b * k, sizeof(int64_t) * k);
      memcpy(out_scores + b * k_fetch, p + off_scores + sizeof(double) * b * k, sizeof(double) * k);
    }
    memcpy(out_counts, p + off_counts, sizeof(int32_t) * B);
    fill_result_tail(out_slots, out_scores, static_cast<int32_t>(B), k_fetch, static_cast<int32_t>(k));
  }
};

}  // namespace impl
}  // namespace rbk

struct rbk_index {
  int dim = 0, dpad = 0, device = 0, sm_count = 0, margin = 16;
  int64_t cap = 0, n_rows = 0, n_live = 0;
  rbk::SlotLayout slot;      // local row -> global slot (rbk_index_set_slot_base; block-cyclic inside a group)
  // The device corpus buffers - rows | inv_norm | norm2 | dead_bits | f64 rows (device tier) - each on its own reserved
  // range, sized for vm_rows rows (the most the device could back); the pointers below are the ranges' bases.
  static constexpr int kVmBuffers = 5;
  rbk::impl::VmRange vm[kVmBuffers];
  int64_t vm_rows = 0;
  size_t vm_gran = 0;        // allocation granularity of the device
  size_t total_mem = 0;      // the device's memory, which sets vm_rows for each storage tier
  uint16_t* rows = nullptr;
  float* inv_norm = nullptr;  // padded to a multiple of kBlockN (+ one tile), NaN-filled
  double* norm2 = nullptr;
  // optional exact-source rows [cap][dim] of x_elem bytes each: float64 (RBK_INDEX_KEEP_F64, x_elem 8) or float32
  // (RBK_INDEX_KEEP_F32, x_elem 4; every stored value is float32-exact, so its widening is the float64 row) or the low
  // halves of float32 rows whose high halves are `rows` (RBK_INDEX_KEEP_F32_SPLIT, x_elem 2; rbk_internal.h); x_elem 0:
  // none
  void* rows_x = nullptr;
  int x_elem = 0;
  bool keep_rows() const { return x_elem != 0; }
  bool f32_rows() const { return x_elem == 4 || x_elem == 2; }   // only float32-exact values may be stored
  size_t x_row_bytes() const { return static_cast<size_t>(dim) * x_elem; }
  // RBK_INDEX_ROWS_ON_HOST: rows_x is pinned, mapped host memory (one pointer under UVA).  Every write to it is
  // stream-ordered: a kernel or copy on `stream`, or the host after a synchronisation of `stream`.
  bool rows_on_host = false;
  // RBK_INDEX_SCAN_F16: `rows` (and the queries' scan copies) hold per-row scaled fp16 instead of bf16, and the scan
  // runs its fp16 instantiation (rbk_scan_f16.cu).  Requires exact rows, so nothing ever decodes these rows as values
  // except the norm kernels: the re-rank, the fallback and the exact scores read rows_x.
  bool scan_f16 = false;
  unsigned int* dead_bits = nullptr;
  int* d_counter = nullptr;   // [0] tombstone counter, [1] eps_c_max (float bits)
  cudaStream_t own_stream = nullptr, stream = nullptr;
  std::mutex mu;
  // ingest staging
  rbk::impl::DevBuf<unsigned char> stage;
  rbk::impl::DevBuf<int64_t> d_slots;
  // compaction scratch: old_to_new, and word prefixes | block sums | chunk prefixes of the liveness scan
  rbk::impl::DevBuf<long long> cp_map;
  rbk::impl::DevBuf<int> cp_scan;
  // search scratch
  rbk::impl::DevBuf<unsigned char> q_raw;
  rbk::impl::DevBuf<uint16_t> q_bf16;
  rbk::impl::DevBuf<double> q_f64, q_norm2, q_eps;
  rbk::impl::DevBuf<float> q_inv_norm, thr_init;
  rbk::impl::DevBuf<unsigned long long> cand;
  rbk::impl::DevBuf<int> cand_cnt, flags, fail_list, part_rows, part_cnt;
  rbk::impl::DevBuf<unsigned int> hist;   // the scan's per-launch scratch (split by fill_scan_params)
  rbk::impl::DevBuf<double> o_scores, part_scores;
  rbk::impl::DevBuf<float> dbg;
  // large-k search scratch (grow-only): theta_q, C_q, emit counters, segment offsets, flat candidate rows + scores
  rbk::impl::DevBuf<float> lg_theta;
  rbk::impl::DevBuf<int> lg_cap, lg_cnt, lg_rows, lg_err;
  rbk::impl::DevBuf<long long> lg_off;
  rbk::impl::DevBuf<double> lg_scores;
  rbk::impl::PinBuf<int> h_lcap, h_lerr;
  rbk::impl::PinBuf<long long> h_loff;
  // segmented sort scratch (grow-only, k_fetch > RBK_MAX_K_FETCH_LARGE only): per-query first run-length slot, the
  // sort's second buffer, run lengths
  rbk::impl::DevBuf<int> ub_toff, ub_rows, ub_len;
  rbk::impl::DevBuf<double> ub_scores;
  rbk::impl::PinBuf<int> h_utoff;
  rbk::impl::DevBuf<unsigned char> o_block;
  rbk::impl::PinBuf<unsigned char> h_block;
  rbk::impl::PinBuf<int> h_flags;
  // rbk_index_search_each_f64: each query's k_fetch (or k_eff) and min_score on the device
  rbk::impl::DevBuf<int> e_k;
  rbk::impl::DevBuf<double> e_min;
  // rbk_index_search_slots_f64: one chunk's local query rows, and the count of tombstoned ones (device, pinned copy)
  rbk::impl::DevBuf<int64_t> sq_rows;
  rbk::impl::DevBuf<int> sq_dead;
  rbk::impl::PinBuf<int> h_sq_dead;
  // rbk_index_similar_pairs_f64: the chunk's corpus map from row pr_r0 on (pr_rows rows; 0: no row can pair), one
  // query group's exact pair counts (device, pinned copy), their offsets and the packed pairs (global slot, score);
  // their copy-back goes to h_block
  CUtensorMap pr_tmap;
  int64_t pr_r0 = 0, pr_rows = 0;
  rbk::impl::DevBuf<int> pr_cnt;
  rbk::impl::DevBuf<long long> pr_off, pr_b;
  rbk::impl::DevBuf<double> pr_s;
  rbk::impl::PinBuf<int> h_pcnt;
  // rbk_index_search_mmr_f64: one query group's packed selection inputs, and its picks (slots | scores); the candidate
  // rows are staged in q_raw
  rbk::impl::DevBuf<unsigned char> mm_in, mm_out;
  CUtensorMap tmap_c;
  int max_lead_tiles = rbk::kMaxLeadTiles;
  int kprime_override = 0;   // > 0 while a batch is re-scanned with the widest candidate margin
  int64_t tmap_c_rows = -1;   // rows the corpus map covers (-1: none); its base, `rows`, moves only in rbk_index_set_tier
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;   // device time of a whole synchronous search
  // scan-kernel timing without a host sync per search: (start, stop) event pairs are resolved lazily
  // (rbk_index_stats, or when the ring wraps) into stats.scan_ms_total / stats.scans_timed
  static constexpr int kTimingRing = 64;
  cudaEvent_t tev[kTimingRing][2] = {};
  uint64_t tev_head = 0, tev_tail = 0;   // [tail, head) pending
  // Small batches (B <= 128, host queries in, host results out) replay ONE captured CUDA graph - H2D of the
  // queries, prep, scan, finalize, D2H of the packed block - instead of paying six API calls per search.  The
  // graph bakes in every pointer and scalar it was captured with: `graph_key` is compared before each replay.
  struct GraphKey {
    const void* ptr[20];
    int64_t n_rows;
    double min_score;
    int B, k_fetch, elem, margin;
    rbk::SlotLayout slot;
    cudaStream_t stream;
  };
  cudaGraphExec_t graph_exec = nullptr;
  GraphKey graph_key;                     // meaningful only while graph_exec != nullptr
  rbk::impl::PinBuf<unsigned char> h_q;   // pinned staging of the queries (the graph's H2D source)
  bool capturing = false;                 // run_scan: no timing events inside a capture
  bool use_graph = true;
  rbk_stats stats;
};


namespace rbk {
namespace impl {

// The per-query cut and threshold of a search_each call, on one index's device (its e_k / e_min, [B]).  Both null in
// every other search, which applies its scalar k_fetch and min_score to every query.
struct QueryCuts {
  const int* k = nullptr;
  const double* min_score = nullptr;
};
// Copies k [B] and min_score [B] from the host into ix->e_k / ix->e_min (caller holds the lock, device current).
rbk_status upload_cuts(rbk_index* ix, int B, const int32_t* k, const double* min_score, QueryCuts* out);
// The argument checks of a search_each call, in check_search_args' order; *K = the largest k (0 when B == 0).
rbk_status check_each_args(rbk_index* ix, int B, bool have_q, int query_dim, const int32_t* k, const double* min_score,
                           int* K);

// A search_slots call works through its slots in chunks of this many queries, each one search, so that its device
// scratch is that of one chunk however many slots it names.
constexpr int kSlotChunk = 1024;
// Enqueues the gather of the stored values of local rows rows[0, B) (host, each < n_rows) into ix->q_raw as float64
// queries, and the copy of the number of tombstoned ones into ix->h_sq_dead[0], which the caller reads after its next
// synchronisation of the stream (caller holds the lock, device current).
rbk_status gather_queries(rbk_index* ix, const int64_t* rows, int B);
// RBK_EINVAL when the last gather met a tombstoned row (after the synchronisation that follows it).
rbk_status check_gathered(const rbk_index* ix);

// rbk_index_search_mmr_f64 and rbk_group_search_mmr_f64.  The argument checks, in the order of check_each_args; *K = the
// largest k (0 when B == 0).
rbk_status check_mmr_args(rbk_index* ix, int B, bool have_q, int query_dim, const int32_t* k, const int32_t* fetch_k,
                          const double* lambda_mult, const double* min_score, const void* out_slots,
                          const void* out_scores, const void* out_counts, int* K);
// The candidate rows of one query group of an MMR call, the stored values of global slots slots[0, n), in two steps:
// host(slots, n) does the host work they need first (outside the timed region), then device(n) enqueues on ix->stream
// what puts them in ix->q_raw as float64 rows [n][dim].
struct MmrStage {
  std::function<rbk_status(const int64_t* slots, int n)> host;
  std::function<rbk_status(int n)> device;
};
// The greedy selection of one chunk of Bc queries of an MMR call (caller holds ix->mu, device current): query b's
// candidates are the first c_counts[b] entries of row b of c_slots / c_scores ([Bc][F], global slots, the search_each
// answer at its fetch_k).  Per contiguous query group whose candidate rows fit kLargeBudget, stage.host, then stage.device put the rows
// in ix->q_raw and launch_mmr_select writes row b of out_slots / out_scores ([Bc][K], host); out_counts[b] = min(k[b],
// c_counts[b]).  check_dead: RBK_ECUDA when the stage's gather (gather_queries) met a tombstoned row, which a candidate
// never is.  *ms_out += the device time from stage.device on (the staging copy or gather, the selection, the copy
// back), which leaves out stage.host's host work.
rbk_status mmr_select_locked(rbk_index* ix, int Bc, int F, const int64_t* c_slots, const double* c_scores,
                             const int32_t* c_counts, const int32_t* k, const double* lambda_mult, int K,
                             const MmrStage& stage, bool check_dead, int64_t* out_slots, double* out_scores,
                             int32_t* out_counts, float* ms_out);

// caller holds ix->mu and has the index's device current.  The scan's query buffer keeps kBlockM zeroed rows beyond
// the last whole query block, so that a scan launch may start at any query (a large-k search's query groups): such a
// launch's query map covers round_up(Bs, kBlockM) rows from its first query.
rbk_status ensure_query_scratch(rbk_index* ix, int B, int elem);
// max_k: RBK_MAX_K_FETCH (the search), RBK_MAX_K_FETCH_LARGE or INT32_MAX (the large-k searches)
rbk_status check_search_args(rbk_index* ix, int B, bool have_q, int query_dim, int k_fetch, double min_score,
                             int max_k = RBK_MAX_K_FETCH);
// Enqueue-only search of device-resident queries: no host synchronisation, exactness flags land in d_flags.
// each: a search_each call's per-query cut and threshold (k_fetch is then the row stride, their largest k).
rbk_status enqueue_search(rbk_index* ix, const void* d_q, int src_type, int B, int k_fetch, double min_score,
                          long long* d_slots, double* d_scores, int* d_counts, int* d_flags,
                          const QueryCuts& each = QueryCuts());
// Synchronous exact search of device-resident queries of `elem` bytes (8 = f64, 4 = f32), retry and exhaustive
// fallback included: rbk_index_search_device for either query type.  Takes the index lock itself.  k_each / min_each
// (host [B], nullable): a search_each call's own cut and threshold per query, k_fetch their largest k.
rbk_status search_device_exact(rbk_index* ix, const void* d_q, int elem, int B, int k_fetch, double min_score,
                               long long* d_slots, double* d_scores, int* d_counts, const int32_t* k_each = nullptr,
                               const double* min_each = nullptr);
// Large-k search of B device-resident f64 queries (caller holds the lock, scratch for B queries is allocated), for
// any k_fetch above the scan's: the count scan, one host synchronisation, then the queries in contiguous groups whose
// device storage fits kLargeBudget, each group costing one emit scan.  `sorted` (the caller's k_fetch is above
// RBK_MAX_K_FETCH_LARGE) picks the cut: the segmented sort in global memory, or one block per query in shared memory.
// k_eff is the number of entries kept per query: min(k_fetch, count()) when sorted, else k_fetch.
//   large_count   : prep, count pass and select per sub-batch at k_eff, then the D2H of C_q (enqueue only);
//   split_by_budget: (after the stream has been synchronised) the groups, from each query's cost in bytes (at least
//                   one query per group);
//   large_prepare : segment offsets (and, sorted, run-length slots) of every query relative to its group, the scratch
//                   for the largest group, zeroed emit and overflow counters (enqueue only);
//   large_emit    : emit scan, exact re-score and cut of the queries [q0, q1) into d_slots / d_scores / d_counts
//                   ([q1 - q0][k_eff]); enqueue only;
//   large_finish  : the D2H of the overflow counter (enqueue only);
//   large_check   : (after the next synchronisation) RBK_ECUDA if any query emitted more rows than its bound.
// A search_each call passes its cuts (each.k: every query's own k_eff) to large_count and large_emit; k_eff is then the
// largest of them: the count scan's running threshold and the row stride of the results.
rbk_status large_count(rbk_index* ix, const void* d_q, int B, int k_eff, double min_score,
                       const QueryCuts& each = QueryCuts());
constexpr int64_t kLargeBudget = 256ll << 20;
// device bytes per candidate: emit row + exact score (sorted in place), and the sort's second buffer
inline int64_t large_cand_bytes(bool sorted) { return sorted ? 4 + 8 + 12 : 4 + 8; }
// device bytes of one query's result in a packed block of k_eff entries (slots, scores, count, flag)
inline int64_t large_result_bytes(int k_eff) { return 16ll * k_eff + 8; }
std::vector<std::pair<int, int>> split_by_budget(const std::vector<int64_t>& cost);
rbk_status large_prepare(rbk_index* ix, int B, bool sorted, const std::vector<std::pair<int, int>>& groups);
rbk_status large_emit(rbk_index* ix, int q0, int q1, bool sorted, int k_eff, double min_score, long long* d_slots,
                      double* d_scores, int* d_counts, const QueryCuts& each = QueryCuts());
rbk_status large_finish(rbk_index* ix);
rbk_status large_check(rbk_index* ix);

// rbk_index_similar_pairs_f64 and rbk_group_similar_pairs_f64.  The argument checks, in the order of the other
// searches, for an index or group answering for global slots [slot_base, slot_base + size).
rbk_status check_pairs_args(int64_t slot_base, int64_t size, double min_score, int64_t first_slot, int64_t max_pairs,
                            const void* out_a, const void* out_b, const void* out_scores, const void* n_out,
                            const void* next_slot);
// The first local row of a shard whose global slot is >= a (n_rows or more when there is none).
int64_t first_row_at(const SlotLayout& s, int64_t a);
// The steps of one chunk of Q <= kSlotChunk queries, the stored rows of global slots [a0, a0 + Q), already float64 in
// ix->q_raw (caller holds the lock, device current, query scratch for Q queries allocated):
//   pairs_count: prep, then the count scan and the threshold-only select over the rows from the tile that holds the
//                first row with a global slot >= a0 on (the triangle), then the D2H of C_q (enqueue only);
//   (after a synchronisation) split_by_budget, and large_prepare(sorted) as for the unbounded search;
//   pairs_emit : emit scan, exact re-score, drop of every pair (a, b) with b <= a, sort and packing of the pairs of the
//                queries [q0, q1), then the D2H of their counts into h_pcnt and of the overflow counter (enqueue only);
//   pairs_fetch: (after a synchronisation) the D2H of the first n packed pairs into h_block: slots [n] | scores [n].
rbk_status pairs_count(rbk_index* ix, int Q, int64_t a0, double min_score);
rbk_status pairs_emit(rbk_index* ix, int q0, int q1, int64_t a0, double min_score);
rbk_status pairs_fetch(rbk_index* ix, int64_t n);
// The paged pass over members `parts` (one index, or a group's members, whose rows together are global slots
// [0 or slot_base, end)), from first_slot on, checked arguments; the caller holds every member's lock.  load(a0, Q)
// enqueues the stored rows of global slots [a0, a0 + Q) into every member's q_raw as float64 queries.  Chunk after
// chunk and query group after query group, every member's packed pairs are counted (one round trip), the rows that
// still fit in max_pairs are copied back (another) and merged per query on the host.  The first row that does not fit
// ends the pass; the rest of its chunk is discarded.  Adds 1 search and *next_slot - first_slot queries to every member.
rbk_status similar_pairs_run(const std::vector<rbk_index*>& parts, int64_t end, double min_score, int64_t first_slot,
                             int64_t max_pairs, const std::function<rbk_status(int64_t, int)>& load, int64_t* out_a,
                             int64_t* out_b, double* out_scores, int64_t* n_out, int64_t* next_slot, float* ms_out);

// The steps of a compaction, shared by rbk_index_compact and rbk_group_compact (caller holds ix->mu and has the index's
// device current).  Staging of C rows, packed: bf16 (or fp16) rows [C][dpad] | exact rows [C][dim] (x_elem bytes each,
// when kept) | norm2 [C] | inv_norm [C].
struct CompactStage {
  uint16_t* rows;
  void* x;
  double* norm2;
  float* inv;
};
int64_t compact_row_bytes(const rbk_index* ix);
// Every allocation of the compaction: the staging of C rows, and the liveness scan's scratch for map chunks of
// chunk_rows rows (a multiple of 32).
rbk_status compact_alloc(rbk_index* ix, int64_t C, int64_t chunk_rows, CompactStage* st);
// Enqueues the liveness scan of rows [0, n_rows): ix->cp_map (each row's rank among the live rows, -1 if tombstoned)
// and its D2H copies: h_chunk_pref [ceil(n_rows / chunk_rows) + 1] (live rows before each map chunk, then all of them)
// and, when h_map is not null, cp_map itself [n_rows].  The caller synchronises the stream.
rbk_status compact_map(rbk_index* ix, int64_t chunk_rows, int* h_chunk_pref, int64_t* h_map);
// Enqueues the packing of the live rows among rows [s0, s0 + n) into staging rows cp_map[s] - rank0.
rbk_status compact_gather(rbk_index* ix, const CompactStage& st, int64_t s0, int64_t n, int64_t rank0);
// Enqueues the reset of rows [n_new, n_rows) to never-appended rows and clears every tombstone bit.
rbk_status compact_tail(rbk_index* ix, int64_t n_new);
// After the stream has been synchronised: the index holds n_new live rows; drops the caches keyed on the corpus.
void compact_commit(rbk_index* ix, int64_t n_new);

// The steps of a storage tier change, shared by rbk_index_set_tier and rbk_group_set_tier (caller holds ix->mu and has
// the index's device current).  tier_prepare makes every allocation the change needs and changes nothing the index
// shows, and checks that a narrowing (float64 to float32 exact rows) changes no stored value (RBK_ENOTF32 otherwise): the
// new exact-row buffer when the rows move or change width - pinned [cap][dim], or a device range mapped for cap rows -
// and, when the row ceiling rises, larger address ranges for buffers 0-3 with their physical chunks mapped there a
// second time.  Then exactly one of tier_abort, which releases what tier_prepare made, or tier_commit, which moves (or
// widens / narrows) the rows, re-derives the scan copy when its type changes, and drops every cache keyed on the old
// tier or the old pointers.  A tier_commit that fails (a CUDA error only) leaves what it has not yet taken over in the
// plan, for tier_abort; the index itself may then be part-way changed.
struct TierPlan {
  uint32_t flags = 0;
  bool move = false, to_host = false, rescan = false;   // move: the exact rows go to a new buffer (to_host: pinned)
  int x_elem = 0;                       // the new exact-row width
  int64_t vm_rows = 0;                  // the ceiling of the new tier
  void* host_rows = nullptr;            // move && to_host: the pinned [cap][dim] buffer
  bool alias[rbk_index::kVmBuffers] = {};
  VmRange vm[rbk_index::kVmBuffers];    // buffers 0-3 re-reserved (where alias[i]); move to the device: buffer 4
  int eps_bits = 0;                     // eps_c_max before the change (float bits)
};
uint32_t index_flags(const rbk_index* ix);
// RBK_EINVAL for a flag set rbk_index_create_ex refuses (check_flags, which it shares), or one the index cannot move to
// (an index with exact rows keeps one of the keep bits, one without gets none; group membership is the caller's).
rbk_status check_flags(uint32_t flags);
rbk_status tier_check(const rbk_index* ix, uint32_t flags);
rbk_status tier_prepare(rbk_index* ix, uint32_t flags, TierPlan* p);
void tier_abort(rbk_index* ix, TierPlan* p);
rbk_status tier_commit(rbk_index* ix, TierPlan* p);
const char* last_error();
// RBK_ENOTF32 (with its message) if any of the n doubles at src - host memory (staged through ix->stage) or, with
// is_device, device memory - is not float32-exact (launch_find_not_f32); changes nothing in the index.  Caller holds
// ix->mu and has the index's device current.
rbk_status check_f32_exact(rbk_index* ix, const double* src, bool is_device, int64_t n);

}  // namespace impl
}  // namespace rbk
