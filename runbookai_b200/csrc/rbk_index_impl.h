// rbk_index_impl.h — the index object behind the opaque `rbk_index*` of include/rbk_knn.h and the host-side
// helpers shared by the two translation units that implement the C ABI: rbk_capi.cu (one index = one GPU) and
// rbk_group.cu (one group = one index per GPU + the NCCL exchange, all behind one call).
#pragma once
#include <mutex>
#include <string>
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

}  // namespace impl
}  // namespace rbk

struct rbk_index {
  int dim = 0, dpad = 0, device = 0, sm_count = 0, margin = 16;
  int64_t cap = 0, n_rows = 0, n_live = 0;
  rbk::SlotLayout slot;      // local row -> global slot (rbk_index_set_slot_base; block-cyclic inside a group)
  uint16_t* rows = nullptr;
  float* inv_norm = nullptr;  // padded to a multiple of kBlockN (+ one tile), NaN-filled
  double* norm2 = nullptr;
  double* rows_f64 = nullptr;   // optional exact-source sidecar [cap][dim] (RBK_INDEX_KEEP_F64)
  bool keep_f64 = false;
  unsigned int* dead_bits = nullptr;
  int* d_counter = nullptr;   // [0] tombstone counter, [1] eps_c_max (float bits)
  cudaStream_t own_stream = nullptr, stream = nullptr;
  std::mutex mu;
  // ingest staging
  rbk::impl::DevBuf<unsigned char> stage;
  rbk::impl::DevBuf<int64_t> d_slots;
  // search scratch
  rbk::impl::DevBuf<unsigned char> q_raw;
  rbk::impl::DevBuf<uint16_t> q_bf16;
  rbk::impl::DevBuf<double> q_f64, q_norm2, q_eps;
  rbk::impl::DevBuf<float> q_inv_norm, thr_init;
  rbk::impl::DevBuf<unsigned long long> cand;
  rbk::impl::DevBuf<int> cand_cnt, flags, fail_list, o_counts, part_rows, part_cnt, maxbin, progress;
  rbk::impl::DevBuf<unsigned int> hist;
  rbk::impl::DevBuf<long long> o_slots;
  rbk::impl::DevBuf<double> o_scores, part_scores;
  rbk::impl::DevBuf<float> dbg;
  rbk::impl::DevBuf<unsigned char> o_block;
  rbk::impl::PinBuf<unsigned char> h_block;
  rbk::impl::PinBuf<int> h_flags, h_counts;
  rbk::impl::PinBuf<long long> h_slots;
  rbk::impl::PinBuf<double> h_scores;
  rbk::impl::PinBuf<float> h_f32;
  CUtensorMap tmap_c;
  int max_lead_tiles = rbk::kMaxLeadTiles;
  int kprime_override = 0;   // > 0 while a batch is re-scanned with the widest candidate margin
  const void* tmap_c_base = nullptr;
  int64_t tmap_c_rows = -1;
  std::vector<cudaEvent_t> ev;
  // scan-kernel timing without a host sync per search: (start, stop) event pairs are resolved lazily
  // (rbk_index_stats, or when the ring wraps) into stats.scan_ms_total / stats.scans_timed
  static constexpr int kTimingRing = 64;
  cudaEvent_t tev[kTimingRing][2] = {};
  uint64_t tev_head = 0, tev_tail = 0;   // [tail, head) pending
  float pending_scan_ms = 0.f;           // scan time of the search being assembled (resolved pairs only)
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

// caller holds ix->mu and has the index's device current
rbk_status ensure_query_scratch(rbk_index* ix, int B, int elem);
rbk_status check_search_args(rbk_index* ix, int B, bool have_q, int query_dim, int k_fetch, double min_score);
// Enqueue-only search of device-resident queries: no host synchronisation, exactness flags land in d_flags.
rbk_status enqueue_search(rbk_index* ix, const void* d_q, int src_type, int B, int k_fetch, double min_score,
                          long long* d_slots, double* d_scores, int* d_counts, int* d_flags);
const char* last_error();

}  // namespace impl
}  // namespace rbk
