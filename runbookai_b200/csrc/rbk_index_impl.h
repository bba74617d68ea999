// rbk_index_impl.h — the index object behind the opaque `rbk_index*` of include/rbk_knn.h and the host-side
// helpers shared by the two translation units that implement the C ABI: rbk_capi.cu (one index = one GPU) and
// rbk_group.cu (one group = one index per GPU + the NCCL exchange, all behind one call).
#pragma once
#include <string.h>

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
// are mapped from `base` on as the index grows and unmapped from the end by rbk_index_trim, so `base` never moves and
// a growth copies nothing.
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
};

// Entries [k_eff, k_fetch) of each of the B result rows of k_fetch entries: slot -1, score NaN (an unbounded search
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
  uint16_t* rows = nullptr;
  float* inv_norm = nullptr;  // padded to a multiple of kBlockN (+ one tile), NaN-filled
  double* norm2 = nullptr;
  double* rows_f64 = nullptr;   // optional exact-source sidecar [cap][dim] (RBK_INDEX_KEEP_F64)
  bool keep_f64 = false;
  // RBK_INDEX_F64_ON_HOST: rows_f64 is pinned, mapped host memory (one pointer under UVA).  Every write to it is
  // stream-ordered: a kernel or copy on `stream`, or the host after a synchronisation of `stream`.
  bool f64_on_host = false;
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
  // unbounded search scratch (grow-only): per-query first run-length slot, the sort's second buffer, run lengths
  rbk::impl::DevBuf<int> ub_toff, ub_rows, ub_len;
  rbk::impl::DevBuf<double> ub_scores;
  rbk::impl::PinBuf<int> h_utoff;
  rbk::impl::DevBuf<unsigned char> o_block;
  rbk::impl::PinBuf<unsigned char> h_block;
  rbk::impl::PinBuf<int> h_flags;
  CUtensorMap tmap_c;
  int max_lead_tiles = rbk::kMaxLeadTiles;
  int kprime_override = 0;   // > 0 while a batch is re-scanned with the widest candidate margin
  int64_t tmap_c_rows = -1;   // rows the corpus map covers (-1: none); its base, `rows`, never moves
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

// caller holds ix->mu and has the index's device current.  slack_rows: zeroed bf16 query rows beyond the last whole
// query block, for callers whose scan launches start at a query that is not a multiple of kBlockM (the unbounded
// search's query groups): such a launch's query map covers round_up(Bs, kBlockM) rows from its first query.
rbk_status ensure_query_scratch(rbk_index* ix, int B, int elem, int slack_rows = 0);
// max_k: RBK_MAX_K_FETCH (the search) or RBK_MAX_K_FETCH_LARGE (the large-k search)
rbk_status check_search_args(rbk_index* ix, int B, bool have_q, int query_dim, int k_fetch, double min_score,
                             int max_k = RBK_MAX_K_FETCH);
// Enqueue-only search of device-resident queries: no host synchronisation, exactness flags land in d_flags.
rbk_status enqueue_search(rbk_index* ix, const void* d_q, int src_type, int B, int k_fetch, double min_score,
                          long long* d_slots, double* d_scores, int* d_counts, int* d_flags);
// Large-k search of B device-resident f64 queries (caller holds the lock, scratch for B queries is allocated), in
// two halves around one host synchronisation of the index stream:
//   large_count: prep, count pass and select per sub-batch, then the D2H of C_q (enqueue only);
//   large_emit : (after the stream has been synchronised) segment offsets on the host, emit pass and exact re-rank
//                per sub-batch into d_slots / d_scores / d_counts, then the D2H of the overflow counter (enqueue only);
//   large_check: (after the next synchronisation) RBK_ECUDA if any query emitted more rows than its bound.
rbk_status large_count(rbk_index* ix, const void* d_q, int B, int k_fetch, double min_score);
rbk_status large_emit(rbk_index* ix, int B, int k_fetch, double min_score, long long* d_slots, double* d_scores,
                      int* d_counts);
rbk_status large_check(rbk_index* ix);

// Unbounded search (k_fetch > RBK_MAX_K_FETCH_LARGE), built on the same count pass: large_count with k_fetch = k_eff,
// one host synchronisation, then the queries in contiguous groups whose device storage fits kUnboundedBudget, each
// group costing one emit scan:
//   split_by_budget   : the groups, from each query's cost in bytes (at least one query per group);
//   unbounded_prepare : segment offsets and run-length slots of every query relative to its group, the scratch for
//                       the largest group, zeroed emit and overflow counters (enqueue only);
//   unbounded_emit    : emit scan, exact re-score and segmented sort of the queries [q0, q1) into d_slots / d_scores /
//                       d_counts ([q1 - q0][k_eff]); enqueue only;
//   unbounded_finish  : the D2H of the overflow counter, for large_check after the next synchronisation.
constexpr int64_t kUnboundedBudget = 256ll << 20;
// device bytes per candidate: emit row + exact score (sorted in place) + the sort's second buffer
constexpr int64_t kUnboundedCandBytes = 4 + 8 + 12;
// device bytes of one query's result in a packed block of k_eff entries (slots, scores, count, flag)
inline int64_t unbounded_result_bytes(int k_eff) { return 16ll * k_eff + 8; }
std::vector<std::pair<int, int>> split_by_budget(const std::vector<int64_t>& cost);
rbk_status unbounded_prepare(rbk_index* ix, int B, const std::vector<std::pair<int, int>>& groups);
rbk_status unbounded_emit(rbk_index* ix, int q0, int q1, int k_eff, double min_score, long long* d_slots,
                          double* d_scores, int* d_counts);
rbk_status unbounded_finish(rbk_index* ix);
const char* last_error();

}  // namespace impl
}  // namespace rbk
