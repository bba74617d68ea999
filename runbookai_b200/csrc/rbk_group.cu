// rbk_group.cu — the multi-GPU index behind ONE handle and ONE call (include/rbk_knn.h, rbk_group_*).
//
// RunbookAI is a single Node process (SURVEY.md §8b/§8e): the deployment that shards a corpus over the GPUs of a
// box is not "one process per GPU under torchrun" (that is bench.py's harness) but one host thread calling
// rbk_group_search_f32.  A group owns one rbk_index per GPU, deals rows out block-cyclically (global slot s lives
// on device (s / block) % G - the index grows at sync time, so no device needs the final corpus size), and answers
// a batch with
//     H2D of the queries to every GPU  ->  the enqueue-only fused scan + finalize on every GPU (its own stream)
//     ->  ONE ncclAllGather of the packed per-GPU blocks (results + exactness flags) over NVLink
//     ->  merge kernel on GPU 0  ->  one D2H, one host synchronisation.
// NCCL is resolved with dlopen("libnccl.so.2") on first use, so the library itself has no link-time dependency on
// it and a one-GPU group never needs it.  A device list that names a device more than once (co-located members, e.g.
// a G-member group on one GPU) has no communicator: member 0's stream waits for each member's block and copies it.
// Exact per-shard fp64 scores make the merge exact; local row order is
// global slot order within a device, so the (score desc, slot asc) tie-break survives (SlotLayout, rbk_internal.h).
#include <dlfcn.h>
#include <nccl.h>   // types and enums only: every NCCL symbol is looked up at run time
#include <string.h>

#include <algorithm>
#include <memory>

#include "rbk_group_plan.h"
#include "rbk_index_impl.h"

using namespace rbk;
using namespace rbk::impl;

namespace {

struct NcclApi {
  void* handle = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  std::string error;
  bool ok = false;
};

NcclApi& nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      api.handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (api.handle) break;
    }
    if (!api.handle) {
      api.error = std::string("NCCL not found (dlopen libnccl.so.2): ") + (dlerror() ? dlerror() : "?");
      return;
    }
    auto sym = [&](const char* n) { return dlsym(api.handle, n); };
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
    api.CommInitAll = reinterpret_cast<decltype(api.CommInitAll)>(sym("ncclCommInitAll"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(sym("ncclAllGather"));
    api.GroupStart = reinterpret_cast<decltype(api.GroupStart)>(sym("ncclGroupStart"));
    api.GroupEnd = reinterpret_cast<decltype(api.GroupEnd)>(sym("ncclGroupEnd"));
    api.ok = api.GetErrorString && api.CommInitAll && api.CommDestroy && api.AllGather && api.GroupStart && api.GroupEnd;
    if (!api.ok) api.error = "libnccl.so.2 lacks a required symbol";
  });
  return api;
}

rbk_status nccl_fail(ncclResult_t r, const char* what) {
  NcclApi& n = nccl_api();
  return fail(RBK_ENCCL, std::string(what) + ": " + (n.GetErrorString ? n.GetErrorString(r) : "NCCL error"));
}
#define NC(expr)                                       \
  do {                                                 \
    ncclResult_t _r = (expr);                          \
    if (_r != ncclSuccess) return nccl_fail(_r, #expr); \
  } while (0)

}  // namespace

struct rbk_group {
  int dim = 0, G = 0;
  int64_t block = 4096;          // rows per placement block
  int64_t n_slots = 0;           // global slots handed out (tombstones included)
  std::vector<int> devices;
  std::vector<rbk_index*> parts;
  std::vector<ncclComm_t> comms; // empty for G == 1 and for a device list with a repeat (co-located members)
  std::mutex mu;
  struct Dev {
    DevBuf<unsigned char> q, local, all;
    cudaEvent_t enqueued = nullptr;   // co-located members: the member's block is written (recorded on its stream)
  };
  std::vector<Dev> dev;
  DevBuf<unsigned char> out;     // device 0: the merged block (dirty_word)
  PinBuf<unsigned char> h_out, h_q;
  PinBuf<double> h_sq;           // rbk_group_search_slots_f64: the members' gathered query rows
  PinBuf<double> h_pq;           // rbk_group_similar_pairs_f64: one chunk's query rows in slot order
  PinBuf<double> h_mm;           // rbk_group_search_mmr_f64: one query group's candidate rows in candidate order
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int64_t redone_batches = 0;
};

namespace {

// global slot -> (device, local row)
inline void locate(const rbk_group* g, int64_t slot, int* dev, int64_t* local) {
  const int64_t blk = slot / g->block;
  *dev = static_cast<int>(blk % g->G);
  *local = (blk / g->G) * g->block + slot % g->block;
}

// RBK_ENOTF32 if the group keeps float32 rows and any of the n rows is not float32-exact (checked on member 0).
rbk_status group_check_f32(rbk_group* g, const double* rows, int64_t n) {
  rbk_index* ix = g->parts[0];
  if (!ix->f32_rows()) return RBK_OK;
  std::lock_guard<std::mutex> lk(ix->mu);
  DeviceGuard dg(ix->device);
  return check_f32_exact(ix, rows, false, n * g->dim);
}

rbk_status group_append(rbk_group* g, const void* rows, int elem, int64_t n, int64_t* first_out) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (n < 0 || (n > 0 && !rows)) return fail(RBK_EINVAL, "bad rows argument");
  std::lock_guard<std::mutex> lk(g->mu);
  if (first_out) *first_out = g->n_slots;
  if (elem == 8) {   // every row of the call, whichever member it would go to, before any member writes
    rbk_status st = group_check_f32(g, static_cast<const double*>(rows), n);
    if (st != RBK_OK) return st;
  }
  const size_t row_bytes = static_cast<size_t>(g->dim) * elem;
  int64_t done = 0;
  while (done < n) {
    const int64_t s = g->n_slots;
    const int64_t take = std::min<int64_t>(n - done, g->block - s % g->block);   // up to the end of this block
    int d;
    int64_t local;
    locate(g, s, &d, &local);
    const unsigned char* src = static_cast<const unsigned char*>(rows) + static_cast<size_t>(done) * row_bytes;
    int64_t first = -1;
    rbk_status st = elem == 8   ? rbk_index_append_f64(g->parts[d], reinterpret_cast<const double*>(src), take, &first)
                    : elem == 4 ? rbk_index_append_f32(g->parts[d], reinterpret_cast<const float*>(src), take, &first)
                                : rbk_index_append_bf16(g->parts[d], reinterpret_cast<const uint16_t*>(src), take, &first);
    if (st != RBK_OK) return st;
    if (first != local) return fail(RBK_EINVAL, "group placement out of step with a member index");
    g->n_slots += take;
    done += take;
  }
  return RBK_OK;
}

// Split global slots (and optionally their rows) by owning device.
void split_slots(const rbk_group* g, const int64_t* slots, int64_t n, std::vector<std::vector<int64_t>>* local,
                 std::vector<std::vector<int64_t>>* order) {
  local->assign(g->G, {});
  if (order) order->assign(g->G, {});
  for (int64_t i = 0; i < n; ++i) {
    int d;
    int64_t l;
    locate(g, slots[i], &d, &l);
    (*local)[d].push_back(l);
    if (order) (*order)[d].push_back(i);
  }
}

// The merged block on device 0 (g->out) is the packed layout with one more word after the flags: the merge kernel
// adds the number of queries some shard could not prove to flags[B].
int64_t dirty_word(const ResultBlock& L) { return L.off_flags + 4 * L.B; }
int64_t merged_bytes(const ResultBlock& L) { return dirty_word(L) + 4; }

// Member d's buffer for the gathered blocks: every member's with NCCL, only member 0's when members are co-located
// (exchange_and_merge copies the blocks there).
bool needs_all(const rbk_group* g, int d) { return g->G > 1 && (d == 0 || !g->comms.empty()); }

// Stages a batch on every device and enqueues its work there: the buffers for the queries and the packed blocks, the
// start event, the H2D of the queries to each device from one pinned copy (so that the G copies run concurrently, one
// per PCIe link), the member's query scratch, then enqueue(d, ix) with the member's lock held and its device current.
// zero_dirty: the caller reads the dirty count, which the merge kernel adds to - start it from zero (its position
// depends on B and k_fetch, so a running count across calls of different shapes would be garbage).
template <typename F>
rbk_status stage_and_enqueue(rbk_group* g, const void* queries, int elem, const ResultBlock& L, bool zero_dirty,
                             F&& enqueue) {
  const int B = static_cast<int>(L.B);
  const size_t q_bytes = static_cast<size_t>(B) * g->dim * elem;
  {
    DeviceGuard dg(g->devices[0]);
    CK(g->h_q.ensure(q_bytes));
    CK(g->h_out.ensure(merged_bytes(L)));
    CK(g->out.ensure(merged_bytes(L)));
    if (zero_dirty) CK(cudaMemsetAsync(g->out.p + dirty_word(L), 0, 4, g->parts[0]->stream));
  }
  memcpy(g->h_q.p, queries, q_bytes);
  for (int d = 0; d < g->G; ++d) {
    rbk_index* ix = g->parts[d];
    std::lock_guard<std::mutex> il(ix->mu);
    DeviceGuard dg(ix->device);
    CK(g->dev[d].q.ensure(q_bytes));
    CK(g->dev[d].local.ensure(L.bytes));
    if (needs_all(g, d)) CK(g->dev[d].all.ensure(L.bytes * g->G));
    if (d == 0) CK(cudaEventRecord(g->ev0, ix->stream));
    CK(cudaMemcpyAsync(g->dev[d].q.p, g->h_q.p, q_bytes, cudaMemcpyHostToDevice, ix->stream));
    rbk_status st = ensure_query_scratch(ix, B, elem);
    if (st != RBK_OK) return st;
    st = enqueue(d, ix);
    if (st != RBK_OK) return st;
  }
  return RBK_OK;
}

// all-gather of the packed blocks (G > 1) + merge on device 0 into g->out; enqueue only.  Co-located members (a device
// list with a repeat, no communicator): member 0's stream waits for every member's block and copies it into its own
// `all` buffer.  k_each (nullable, on device 0): query b is cut at k_each[b], k_fetch being the row stride.
rbk_status exchange_and_merge(rbk_group* g, const ResultBlock& L, int k_fetch, const int* k_each = nullptr) {
  if (g->G > 1 && g->comms.empty()) {
    for (int d = 1; d < g->G; ++d) {
      DeviceGuard dg(g->devices[d]);
      CK(cudaEventRecord(g->dev[d].enqueued, g->parts[d]->stream));
    }
    DeviceGuard dg(g->devices[0]);
    cudaStream_t s0 = g->parts[0]->stream;
    for (int d = 0; d < g->G; ++d) {
      if (d > 0) CK(cudaStreamWaitEvent(s0, g->dev[d].enqueued, 0));
      // Member d writes its block again (the next call, query group or re-answer) only after collect() has
      // synchronised s0, which orders that write after this copy: a change that drops that synchronisation must make
      // member d's stream wait for the copy instead.
      CK(cudaMemcpyAsync(g->dev[0].all.p + d * L.bytes, g->dev[d].local.p, L.bytes, cudaMemcpyDefault, s0));
    }
  } else if (g->G > 1) {
    NcclApi& n = nccl_api();
    NC(n.GroupStart());
    for (int d = 0; d < g->G; ++d) {
      ncclResult_t r = n.AllGather(g->dev[d].local.p, g->dev[d].all.p, L.bytes, ncclUint8, g->comms[d],
                                   g->parts[d]->stream);
      if (r != ncclSuccess) {
        n.GroupEnd();
        return nccl_fail(r, "ncclAllGather");
      }
    }
    NC(n.GroupEnd());
  }
  DeviceGuard dg(g->devices[0]);
  const char* base = reinterpret_cast<const char*>(g->G > 1 ? g->dev[0].all.p : g->dev[0].local.p);
  unsigned char* o = g->out.p;
  CK(launch_merge_shards(g->G, static_cast<int>(L.B), k_fetch, base, base + L.off_scores, base + L.off_counts,
                         base + L.off_flags, L.bytes, L.bytes, L.bytes, L.bytes, L.slots(o), L.scores(o), L.counts(o),
                         L.flags(o), g->parts[0]->stream, k_each));
  return RBK_OK;
}

// D2H of the merged block, the stop event and the host round trip on device 0.
rbk_status collect(rbk_group* g, const ResultBlock& L) {
  rbk_index* i0 = g->parts[0];
  DeviceGuard dg(i0->device);
  CK(cudaMemcpyAsync(g->h_out.p, g->out.p, merged_bytes(L), cudaMemcpyDeviceToHost, i0->stream));
  CK(cudaEventRecord(g->ev1, i0->stream));
  CK(cudaStreamSynchronize(i0->stream));
  return RBK_OK;
}

// k_each / min_each (host [B], nullable; checked by the caller): a search_each call's cut and threshold per query,
// k_fetch their largest k.  Every member gets them on its own device; the merge reads member 0's copy.
// group_search_locked: the caller holds g->mu and has checked the arguments (B > 0).
rbk_status group_search_locked(rbk_group* g, const void* queries, int elem, int32_t B, int32_t k_fetch,
                               double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                               float* ms_out, const int32_t* k_each = nullptr, const double* min_each = nullptr) {
  rbk_status st;
  const ResultBlock L(B, k_fetch);
  const int src_type = elem == 8 ? 0 : 1;
  const int* merge_k = nullptr;
  st = stage_and_enqueue(g, queries, elem, L, /*zero_dirty=*/true, [&](int d, rbk_index* ix) {
    unsigned char* l = g->dev[d].local.p;
    QueryCuts each;
    if (k_each) {
      rbk_status s2 = upload_cuts(ix, B, k_each, min_each, &each);
      if (s2 != RBK_OK) return s2;
      if (d == 0) merge_k = each.k;
    }
    return enqueue_search(ix, g->dev[d].q.p, src_type, B, k_fetch, min_score, L.slots(l), L.scores(l), L.counts(l),
                          L.flags(l), each);
  });
  if (st != RBK_OK) return st;
  st = exchange_and_merge(g, L, k_fetch, merge_k);
  if (st != RBK_OK) return st;
  st = collect(g, L);   // the ONE host round trip of an exact batch
  if (st != RBK_OK) return st;
  int dirty_total = 0;
  memcpy(&dirty_total, g->h_out.p + dirty_word(L), 4);
  if (dirty_total != 0) {
    // some shard could not prove a query (more near-ties than its candidate margin): every shard re-answers the
    // batch through the synchronous path (wide rescan, then the exhaustive fp64 kernel), and the exchange is redone
    g->redone_batches++;
    for (int d = 0; d < g->G; ++d) {
      unsigned char* l = g->dev[d].local.p;
      // the staged queries keep the caller's type: f64 ones must not be read as f32
      st = search_device_exact(g->parts[d], g->dev[d].q.p, elem, B, k_fetch, min_score, L.slots(l), L.scores(l),
                               L.counts(l), k_each, min_each);
      if (st != RBK_OK) return st;
      DeviceGuard dg(g->parts[d]->device);
      CK(cudaMemsetAsync(L.flags(l), 0, static_cast<size_t>(B) * 4, g->parts[d]->stream));   // exact by construction
    }
    st = exchange_and_merge(g, L, k_fetch, merge_k);   // (the re-answer re-uploaded the same cuts in place)
    if (st != RBK_OK) return st;
    st = collect(g, L);
    if (st != RBK_OK) return st;
  }
  if (ms_out) cudaEventElapsedTime(ms_out, g->ev0, g->ev1);
  L.unpack(g->h_out.p, out_slots, out_scores, out_counts);
  return RBK_OK;
}

rbk_status group_search(rbk_group* g, const void* queries, int elem, int32_t B, int32_t query_dim, int32_t k_fetch,
                        double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts, float* ms_out,
                        const int32_t* k_each = nullptr, const double* min_each = nullptr) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  rbk_status st = check_search_args(g->parts[0], B, queries != nullptr, query_dim, k_fetch, min_score);
  if (st != RBK_OK) return st;
  if (ms_out) *ms_out = 0.f;
  if (B == 0) return RBK_OK;
  std::lock_guard<std::mutex> lk(g->mu);
  return group_search_locked(g, queries, elem, B, k_fetch, min_score, out_slots, out_scores, out_counts, ms_out, k_each,
                             min_each);
}

// Large-k search over the group, k_fetch in [1, max_k] (the pipeline and the k_eff / cut rule of rbk_index_impl.h):
// the count scan on every device and ONE wait for all of them, then the queries in contiguous groups whose candidates
// on all devices together, plus the result blocks they move, fit kLargeBudget.  Per query group: emit scan, exact
// re-score and cut on every device into its packed block of k_eff entries per query (flags zero: the answers are
// exact by construction), the all-gather and merge of group_search, and the copy into the caller's rows of k_fetch
// entries.
// k_each / min_each: as for group_search; each query is cut at its own k_eff (by the same rule, from the group's count).
// group_search_large_locked: the caller holds g->mu and has checked the arguments (B > 0).
rbk_status group_search_large_locked(rbk_group* g, const double* queries, int32_t B, int32_t k_fetch, double min_score,
                                     int64_t* out_slots, double* out_scores, int32_t* out_counts, float* ms_out,
                                     const int32_t* k_each = nullptr, const double* min_each = nullptr) {
  rbk_status st;
  const bool sorted = k_fetch > RBK_MAX_K_FETCH_LARGE;
  const int k_eff = sorted ? static_cast<int>(std::min<int64_t>(k_fetch, rbk_group_count(g))) : k_fetch;
  if (k_eff == 0) {
    fill_result_tail(out_slots, out_scores, B, k_fetch, 0);
    memset(out_counts, 0, sizeof(int32_t) * B);
    return RBK_OK;
  }
  std::vector<int32_t> k_eff_each;
  if (k_each)
    for (int b = 0; b < B; ++b)
      k_eff_each.push_back(sorted ? static_cast<int32_t>(std::min<int64_t>(k_each[b], rbk_group_count(g))) : k_each[b]);
  std::vector<QueryCuts> each(g->G);   // every member's copy of the cuts, on its own device
  st = stage_and_enqueue(g, queries, 8, ResultBlock(B, 1), /*zero_dirty=*/false, [&](int d, rbk_index* ix) {
    if (k_each) {
      rbk_status s2 = upload_cuts(ix, B, k_eff_each.data(), min_each, &each[d]);
      if (s2 != RBK_OK) return s2;
    }
    return large_count(ix, g->dev[d].q.p, B, k_eff, min_score, each[d]);
  });
  if (st != RBK_OK) return st;
  for (int d = 0; d < g->G; ++d) {
    DeviceGuard dg(g->parts[d]->device);
    CK(cudaStreamSynchronize(g->parts[d]->stream));
  }
  // a query's cost: its candidates on every device, and its result in the local block, the all-gathered blocks and
  // the merged block
  std::vector<int64_t> cost(B);
  for (int b = 0; b < B; ++b) {
    cost[b] = (g->G + 2) * large_result_bytes(k_eff);
    for (rbk_index* ix : g->parts) cost[b] += ix->h_lcap.p[b] * large_cand_bytes(sorted);
  }
  const std::vector<std::pair<int, int>> groups = split_by_budget(cost);
  int max_group = 0;
  for (const auto& gr : groups) max_group = std::max(max_group, gr.second - gr.first);
  const ResultBlock Lmax(max_group, k_eff);
  {
    DeviceGuard dg(g->devices[0]);
    CK(g->h_out.ensure(merged_bytes(Lmax)));
    CK(g->out.ensure(merged_bytes(Lmax)));
  }
  for (int d = 0; d < g->G; ++d) {
    rbk_index* ix = g->parts[d];
    std::lock_guard<std::mutex> il(ix->mu);
    DeviceGuard dg(ix->device);
    CK(g->dev[d].local.ensure(Lmax.bytes));
    if (needs_all(g, d)) CK(g->dev[d].all.ensure(Lmax.bytes * g->G));
    st = large_prepare(ix, B, sorted, groups);
    if (st != RBK_OK) return st;
  }
  for (const auto& gr : groups) {
    const int Bg = gr.second - gr.first;
    const ResultBlock L(Bg, k_eff);
    for (int d = 0; d < g->G; ++d) {
      rbk_index* ix = g->parts[d];
      std::lock_guard<std::mutex> il(ix->mu);
      DeviceGuard dg(ix->device);
      unsigned char* l = g->dev[d].local.p;
      st = large_emit(ix, gr.first, gr.second, sorted, k_eff, min_score, L.slots(l), L.scores(l), L.counts(l),
                      each[d]);
      if (st == RBK_OK && gr.second == B) st = large_finish(ix);   // the overflow count rides the last round trip
      if (st != RBK_OK) return st;
      CK(cudaMemsetAsync(L.flags(l), 0, static_cast<size_t>(Bg) * 4, ix->stream));
    }
    st = exchange_and_merge(g, L, k_eff, each[0].k ? each[0].k + gr.first : nullptr);   // the group's own rows
    if (st != RBK_OK) return st;
    st = collect(g, L);
    if (st != RBK_OK) return st;
    const size_t o = static_cast<size_t>(gr.first) * k_fetch;
    L.unpack_rows(g->h_out.p, k_fetch, out_slots + o, out_scores + o, out_counts + gr.first);
  }
  for (int d = 0; d < g->G; ++d) {   // every device's overflow counter has landed on the host
    if (d > 0) {                     // (collect has waited for device 0)
      DeviceGuard dg(g->parts[d]->device);
      CK(cudaStreamSynchronize(g->parts[d]->stream));
    }
    st = large_check(g->parts[d]);
    if (st != RBK_OK) return st;
  }
  if (ms_out) cudaEventElapsedTime(ms_out, g->ev0, g->ev1);
  return RBK_OK;
}

rbk_status group_search_large(rbk_group* g, const double* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                              double min_score, int max_k, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                              float* ms_out, const int32_t* k_each = nullptr, const double* min_each = nullptr) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  rbk_status st = check_search_args(g->parts[0], B, queries != nullptr, query_dim, k_fetch, min_score, max_k);
  if (st != RBK_OK) return st;
  if (ms_out) *ms_out = 0.f;
  if (B == 0) return RBK_OK;
  std::lock_guard<std::mutex> lk(g->mu);
  return group_search_large_locked(g, queries, B, k_fetch, min_score, out_slots, out_scores, out_counts, ms_out, k_each,
                                   min_each);
}

// The stored values of global slots slots[0, B) (each < n_slots) as float64 queries into q [B][dim]: every member
// gathers the rows it holds into its query scratch and copies them into the pinned staging g->h_sq, one wait per member,
// which also brings back its count of tombstoned rows (RBK_EINVAL if any).  Caller holds g->mu.
rbk_status group_gather_locked(rbk_group* g, const int64_t* slots, int B, double* q, bool allow_dead);
rbk_status group_gather(rbk_group* g, const int64_t* slots, int B, double* q) {
  std::vector<std::unique_lock<std::mutex>> locks;
  for (rbk_index* ix : g->parts) locks.emplace_back(ix->mu);
  return group_gather_locked(g, slots, B, q, /*allow_dead=*/false);
}

// group_gather with every member's lock held by the caller.  allow_dead: a tombstoned slot is not refused; its query
// is zeros (launch_gather_rows).
rbk_status group_gather_locked(rbk_group* g, const int64_t* slots, int B, double* q, bool allow_dead) {
  std::vector<std::vector<int64_t>> local, order;
  split_slots(g, slots, B, &local, &order);
  {
    DeviceGuard dg(g->devices[0]);
    CK(g->h_sq.ensure(static_cast<size_t>(B) * g->dim));
  }
  size_t first = 0;   // member d's rows land at h_sq rows [first, first + n) in member order
  for (int d = 0; d < g->G; ++d) {
    const int n = static_cast<int>(local[d].size());
    if (n == 0) continue;
    rbk_index* ix = g->parts[d];
    DeviceGuard dg(ix->device);
    rbk_status st = gather_queries(ix, local[d].data(), n);
    if (st != RBK_OK) return st;
    CK(cudaMemcpyAsync(g->h_sq.p + first * g->dim, ix->q_raw.p, sizeof(double) * n * g->dim, cudaMemcpyDeviceToHost,
                       ix->stream));
    first += n;
  }
  first = 0;
  for (int d = 0; d < g->G; ++d) {
    const int n = static_cast<int>(local[d].size());
    if (n == 0) continue;
    rbk_index* ix = g->parts[d];
    DeviceGuard dg(ix->device);
    CK(cudaStreamSynchronize(ix->stream));
    rbk_status st = allow_dead ? RBK_OK : check_gathered(ix);
    if (st != RBK_OK) return st;
    for (int i = 0; i < n; ++i)
      memcpy(q + static_cast<size_t>(order[d][i]) * g->dim, g->h_sq.p + (first + i) * g->dim, sizeof(double) * g->dim);
    first += n;
  }
  return RBK_OK;
}

// One compaction's events, one pair per member; destroyed on every return.
struct CompactEvents {
  std::vector<cudaEvent_t> gathered, copied;
  explicit CompactEvents(int G) : gathered(G, nullptr), copied(G, nullptr) {}
  ~CompactEvents() {
    for (cudaEvent_t e : gathered)
      if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : copied)
      if (e) cudaEventDestroy(e);
  }
};

// rbk_group_compact: the plan of rbk_group_plan.h, run chunk by chunk.  Every member packs its survivors of the chunk
// into its own staging (the gather kernel of rbk_index_compact) and records `gathered`; every receiver waits for the
// senders it reads, copies their segments into its own rows on its own stream and records `copied`; a sender waits for
// the receivers that read its staging before it refills it.
rbk_status group_compact(rbk_group* g, int64_t* old_to_new, int64_t old_to_new_len) {
  if (!g) return fail(RBK_EINVAL, "null group");
  std::lock_guard<std::mutex> lk(g->mu);
  const int G = g->G;
  const int64_t n = g->n_slots, block = g->block;
  if (old_to_new && old_to_new_len < n) return fail(RBK_EINVAL, "old_to_new_len is shorter than rbk_group_size()");
  std::vector<std::unique_lock<std::mutex>> member_locks;
  member_locks.reserve(G);
  for (rbk_index* ix : g->parts) member_locks.emplace_back(ix->mu);
  int64_t n_live = 0;
  for (int d = 0; d < G; ++d) {
    if (g->parts[d]->n_rows != group_plan::member_rows(G, block, n, d))
      return fail(RBK_EINVAL, "group placement out of step with a member index");
    n_live += g->parts[d]->n_live;
  }
  if (n_live == n) {   // no tombstones (or an empty group): nothing moves
    for (int64_t s = 0; old_to_new && s < n; ++s) old_to_new[s] = s;
    return RBK_OK;
  }
  // A member stages whole blocks, 64 MB of packed rows or one block if that is more; a chunk is R rounds of G blocks,
  // so that each member's share of it is at most R blocks of consecutive local rows.
  const int64_t R = std::max<int64_t>(1, (64ll << 20) / (block * compact_row_bytes(g->parts[0])));
  // every allocation before the first row moves: RBK_ENOMEM leaves the group untouched
  std::vector<CompactStage> stage(G);
  std::vector<std::vector<int>> pref(G);
  std::vector<std::vector<int64_t>> local_map(G);
  std::vector<int> eps(G, 0);
  CompactEvents ev(G);
  for (int d = 0; d < G; ++d) {
    rbk_index* ix = g->parts[d];
    DeviceGuard dg(ix->device);
    rbk_status st = compact_alloc(ix, R * block, block, &stage[d]);
    if (st != RBK_OK) return st;
    CK(cudaEventCreateWithFlags(&ev.gathered[d], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&ev.copied[d], cudaEventDisableTiming));
    pref[d].assign(static_cast<size_t>((ix->n_rows + block - 1) / block + 1), 0);
    if (old_to_new) local_map[d].resize(static_cast<size_t>(ix->n_rows));
  }
  // 1. Map: each member's liveness scan, per-block survivor counts (map chunk = one block) and its eps_c_max.
  for (int d = 0; d < G; ++d) {
    rbk_index* ix = g->parts[d];
    DeviceGuard dg(ix->device);
    if (ix->n_rows > 0) {
      rbk_status st = compact_map(ix, block, pref[d].data(), old_to_new ? local_map[d].data() : nullptr);
      if (st != RBK_OK) return st;
    }
    CK(cudaMemcpyAsync(&eps[d], ix->d_counter + 1, sizeof(int), cudaMemcpyDeviceToHost, ix->stream));
  }
  for (int d = 0; d < G; ++d) {
    DeviceGuard dg(g->parts[d]->device);
    CK(cudaStreamSynchronize(g->parts[d]->stream));
  }
  for (int d = 0; d < G; ++d)
    if (pref[d].back() != g->parts[d]->n_live)
      return fail(RBK_ECUDA, "compaction: the tombstone bits of device " + std::to_string(g->devices[d]) + " count " +
                                 std::to_string(pref[d].back()) + " live rows, its index " +
                                 std::to_string(g->parts[d]->n_live) + " (the group was not changed)");
  const int64_t nb = (n + block - 1) / block;
  std::vector<int64_t> block_live(static_cast<size_t>(nb));
  for (int64_t b = 0; b < nb; ++b) {
    const std::vector<int>& p = pref[b % G];
    block_live[b] = p[b / G + 1] - p[b / G];
  }
  // 2. Plan, and the caller's map: a survivor's new slot is its block's base plus its rank within the block.
  const group_plan::Plan plan = group_plan::make_plan(G, block, n, block_live, R * G);
  if (old_to_new) {
    std::vector<const int64_t*> rank(G);
    std::vector<const int*> block_pref(G);
    for (int d = 0; d < G; ++d) {
      rank[d] = local_map[d].data();
      block_pref[d] = pref[d].data();
    }
    group_plan::fill_old_to_new(G, block, n, plan, rank, block_pref, old_to_new);
  }
  // A moved row carries its share of the corpus-side error bound (and the off-band marker) to its new device: every
  // member takes the largest, which only widens the bound.
  const int eps_max = *std::max_element(eps.begin(), eps.end());   // non-negative floats order like ints
  // Peer access makes the cross-device copies direct; without it they are still correct, staged by the driver.
  for (int d = 0; d < G; ++d)
    for (int e = 0; e < G; ++e) {
      int can = 0;
      if (g->devices[d] == g->devices[e] ||   // co-located members: no peer to enable
          cudaDeviceCanAccessPeer(&can, g->devices[d], g->devices[e]) != cudaSuccess || !can)
        continue;
      DeviceGuard dg(g->devices[d]);
      if (cudaDeviceEnablePeerAccess(g->devices[e], 0) != cudaSuccess) cudaGetLastError();   // already enabled
    }
  cudaGetLastError();
  // 3. Move.  pending[e][r]: receiver r has read e's staging since e's last gather.
  std::vector<std::vector<char>> pending(G, std::vector<char>(G, 0));
  for (const group_plan::Chunk& c : plan.chunks) {
    for (int e = 0; e < G; ++e) {
      if (c.staged[e] == 0) continue;
      rbk_index* ix = g->parts[e];
      DeviceGuard dg(ix->device);
      for (int r = 0; r < G; ++r)
        if (pending[e][r]) {
          CK(cudaStreamWaitEvent(ix->stream, ev.copied[r], 0));
          pending[e][r] = 0;
        }
      rbk_status st = compact_gather(ix, stage[e], c.g0[e], c.gn[e], c.rank0[e]);
      if (st != RBK_OK) return st;
      CK(cudaEventRecord(ev.gathered[e], ix->stream));
    }
    for (int d = 0; d < G; ++d) {
      rbk_index* ix = g->parts[d];
      DeviceGuard dg(ix->device);
      std::vector<char> waited(G, 0);
      bool wrote = false;
      for (const group_plan::Segment& s : c.segs) {
        if (s.dst != d) continue;
        if (s.src != d && !waited[s.src]) {
          CK(cudaStreamWaitEvent(ix->stream, ev.gathered[s.src], 0));
          waited[s.src] = 1;
        }
        const CompactStage& ss = stage[s.src];
        // device, peer or mapped host rows (RBK_INDEX_F64_ON_HOST): UVA picks the direction
        CK(cudaMemcpyAsync(ix->rows + s.dst_row * ix->dpad, ss.rows + s.src_off * ix->dpad,
                           static_cast<size_t>(s.len) * ix->dpad * 2, cudaMemcpyDefault, ix->stream));
        if (ix->keep_rows())   // moved as bytes, x_row_bytes() per row
          CK(cudaMemcpyAsync(static_cast<unsigned char*>(ix->rows_x) + s.dst_row * ix->x_row_bytes(),
                             static_cast<const unsigned char*>(ss.x) + s.src_off * ix->x_row_bytes(),
                             static_cast<size_t>(s.len) * ix->x_row_bytes(), cudaMemcpyDefault, ix->stream));
        CK(cudaMemcpyAsync(ix->norm2 + s.dst_row, ss.norm2 + s.src_off, static_cast<size_t>(s.len) * 8,
                           cudaMemcpyDefault, ix->stream));
        CK(cudaMemcpyAsync(ix->inv_norm + s.dst_row, ss.inv + s.src_off, static_cast<size_t>(s.len) * 4,
                           cudaMemcpyDefault, ix->stream));
        wrote = true;
      }
      if (!wrote) continue;
      CK(cudaEventRecord(ev.copied[d], ix->stream));
      for (int e = 0; e < G; ++e)
        if (waited[e]) pending[e][d] = 1;
    }
  }
  // 4. Finish: every member holds the slots below n_live that the layout gives it.
  for (int d = 0; d < G; ++d) {
    rbk_index* ix = g->parts[d];
    DeviceGuard dg(ix->device);
    rbk_status st = compact_tail(ix, group_plan::member_rows(G, block, n_live, d));
    if (st != RBK_OK) return st;
    CK(cudaMemcpyAsync(ix->d_counter + 1, &eps_max, sizeof(int), cudaMemcpyHostToDevice, ix->stream));
  }
  for (int d = 0; d < G; ++d) {
    rbk_index* ix = g->parts[d];
    DeviceGuard dg(ix->device);
    CK(cudaStreamSynchronize(ix->stream));
    compact_commit(ix, group_plan::member_rows(G, block, n_live, d));
  }
  g->n_slots = n_live;
  return RBK_OK;
}

}  // namespace

extern "C" {

rbk_status rbk_group_create(int32_t dim, const int32_t* device_ids, int32_t n_devices, int64_t capacity_hint,
                            uint32_t flags, rbk_group** out) {
  if (!out) return fail(RBK_EINVAL, "out is null");
  *out = nullptr;
  if (!device_ids || n_devices < 1 || n_devices > 64) return fail(RBK_EINVAL, "bad device list");
  bool repeat = false;   // NCCL refuses two ranks on one device: such a group exchanges its blocks by copies
  for (int a = 0; a < n_devices; ++a)
    for (int b = a + 1; b < n_devices; ++b) repeat = repeat || device_ids[a] == device_ids[b];
  std::unique_ptr<rbk_group> g(new (std::nothrow) rbk_group());
  if (!g) return fail(RBK_ENOMEM, "out of host memory");
  g->dim = dim;
  g->G = n_devices;
  g->devices.assign(device_ids, device_ids + n_devices);
  g->dev.resize(n_devices);
  auto destroy_parts = [&]() {
    for (rbk_index* ix : g->parts) rbk_index_destroy(ix);
    g->parts.clear();
  };
  for (int d = 0; d < n_devices; ++d) {
    rbk_index* ix = nullptr;
    rbk_status st = rbk_index_create_ex(dim, device_ids[d], capacity_hint / n_devices + g->block, flags, &ix);
    if (st != RBK_OK) {
      destroy_parts();
      return st;
    }
    ix->slot.block = static_cast<int32_t>(g->block);
    ix->slot.G = n_devices;
    ix->slot.g = d;
    g->parts.push_back(ix);
  }
  if (n_devices > 1 && !repeat) {
    NcclApi& n = nccl_api();
    if (!n.ok) {
      destroy_parts();
      return fail(RBK_ENCCL, n.error + " (a group of more than one GPU exchanges its per-GPU lists with ncclAllGather)");
    }
    g->comms.resize(n_devices);
    ncclResult_t r = n.CommInitAll(g->comms.data(), n_devices, g->devices.data());
    if (r != ncclSuccess) {
      g->comms.clear();
      destroy_parts();
      return nccl_fail(r, "ncclCommInitAll");
    }
  }
  {
    DeviceGuard dg(g->devices[0]);
    if (cudaEventCreate(&g->ev0) != cudaSuccess || cudaEventCreate(&g->ev1) != cudaSuccess) {
      rbk_group_destroy(g.release());
      return fail(RBK_ECUDA, "cudaEventCreate");
    }
  }
  for (int d = 1; repeat && d < n_devices; ++d) {
    DeviceGuard dg(g->devices[d]);
    if (cudaEventCreateWithFlags(&g->dev[d].enqueued, cudaEventDisableTiming) != cudaSuccess) {
      rbk_group_destroy(g.release());
      return fail(RBK_ECUDA, "cudaEventCreate");
    }
  }
  *out = g.release();
  return RBK_OK;
}

void rbk_group_destroy(rbk_group* g) {
  if (!g) return;
  for (size_t d = 0; d < g->parts.size(); ++d) {
    DeviceGuard dg(g->devices[d]);
    if (g->parts[d] && g->parts[d]->stream) cudaStreamSynchronize(g->parts[d]->stream);
    g->dev[d].q.release();
    g->dev[d].local.release();
    g->dev[d].all.release();
    if (g->dev[d].enqueued) cudaEventDestroy(g->dev[d].enqueued);
  }
  if (!g->comms.empty()) {
    NcclApi& n = nccl_api();
    for (ncclComm_t c : g->comms)
      if (c && n.CommDestroy) n.CommDestroy(c);
  }
  if (!g->devices.empty()) {
    DeviceGuard dg(g->devices[0]);
    g->out.release();
    g->h_out.release();
    g->h_q.release();
    g->h_sq.release();
    g->h_pq.release();
    g->h_mm.release();
    if (g->ev0) cudaEventDestroy(g->ev0);
    if (g->ev1) cudaEventDestroy(g->ev1);
  }
  for (rbk_index* ix : g->parts) rbk_index_destroy(ix);
  delete g;
}

rbk_status rbk_group_append_f64(rbk_group* g, const double* rows, int64_t n, int64_t* first) {
  return group_append(g, rows, 8, n, first);
}
rbk_status rbk_group_append_f32(rbk_group* g, const float* rows, int64_t n, int64_t* first) {
  return group_append(g, rows, 4, n, first);
}
rbk_status rbk_group_append_bf16(rbk_group* g, const uint16_t* rows, int64_t n, int64_t* first) {
  return group_append(g, rows, 2, n, first);
}

rbk_status rbk_group_overwrite_f64_batch(rbk_group* g, const int64_t* slots, int64_t n, const double* rows) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (n < 0 || (n > 0 && (!slots || !rows))) return fail(RBK_EINVAL, "bad argument");
  std::lock_guard<std::mutex> lk(g->mu);
  for (int64_t i = 0; i < n; ++i)
    if (slots[i] < 0 || slots[i] >= g->n_slots) return fail(RBK_EINVAL, "slot out of range");
  rbk_status worst = group_check_f32(g, rows, n);   // no member writes if any row is refused
  if (worst != RBK_OK) return worst;
  std::vector<std::vector<int64_t>> local, order;
  split_slots(g, slots, n, &local, &order);
  std::string msg;
  for (int d = 0; d < g->G; ++d) {
    if (local[d].empty()) continue;
    std::vector<double> part(local[d].size() * static_cast<size_t>(g->dim));
    for (size_t i = 0; i < order[d].size(); ++i)
      memcpy(&part[i * g->dim], rows + static_cast<size_t>(order[d][i]) * g->dim, sizeof(double) * g->dim);
    rbk_status st = rbk_index_overwrite_f64_batch(g->parts[d], local[d].data(), static_cast<int64_t>(local[d].size()),
                                                  part.data());
    if (st != RBK_OK) {   // keep going: the live slots of the other devices are still written, as within one index
      worst = st;
      msg = last_error();
    }
  }
  return worst == RBK_OK ? RBK_OK : fail(worst, msg);
}

rbk_status rbk_group_tombstone(rbk_group* g, const int64_t* slots, int64_t n) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (n < 0 || (n > 0 && !slots)) return fail(RBK_EINVAL, "bad slots argument");
  std::lock_guard<std::mutex> lk(g->mu);
  for (int64_t i = 0; i < n; ++i)
    if (slots[i] < 0 || slots[i] >= g->n_slots) return fail(RBK_EINVAL, "slot out of range");
  std::vector<std::vector<int64_t>> local;
  split_slots(g, slots, n, &local, nullptr);
  for (int d = 0; d < g->G; ++d) {
    if (local[d].empty()) continue;
    rbk_status st = rbk_index_tombstone(g->parts[d], local[d].data(), static_cast<int64_t>(local[d].size()));
    if (st != RBK_OK) return st;
  }
  return RBK_OK;
}

rbk_status rbk_group_clear(rbk_group* g) {
  if (!g) return fail(RBK_EINVAL, "null group");
  std::lock_guard<std::mutex> lk(g->mu);
  for (rbk_index* ix : g->parts) {
    rbk_status st = rbk_index_clear(ix);
    if (st != RBK_OK) return st;
  }
  g->n_slots = 0;
  return RBK_OK;
}

rbk_status rbk_group_trim(rbk_group* g) {
  if (!g) return fail(RBK_EINVAL, "null group");
  std::lock_guard<std::mutex> lk(g->mu);
  for (rbk_index* ix : g->parts) {   // synchronises each member's stream, which the group's searches run on
    rbk_status st = rbk_index_trim(ix);
    if (st != RBK_OK) return st;
  }
  for (size_t d = 0; d < g->parts.size(); ++d) {
    DeviceGuard dg(g->devices[d]);
    g->dev[d].q.release();
    g->dev[d].local.release();
    g->dev[d].all.release();
  }
  DeviceGuard dg(g->devices[0]);
  g->out.release();
  g->h_out.release();
  g->h_q.release();
  g->h_sq.release();
  g->h_pq.release();
  g->h_mm.release();
  return RBK_OK;
}

rbk_status rbk_group_compact(rbk_group* g, int64_t* old_to_new, int64_t old_to_new_len) {
  return group_compact(g, old_to_new, old_to_new_len);
}

// rbk_index_set_tier on every member: every member's allocations (tier_prepare) before any member changes, as
// rbk_group_compact allocates before the first row moves.
rbk_status rbk_group_set_tier(rbk_group* g, uint32_t flags) {
  if (!g) return fail(RBK_EINVAL, "null group");
  std::lock_guard<std::mutex> lk(g->mu);
  std::vector<std::unique_lock<std::mutex>> member_locks;
  member_locks.reserve(g->G);
  for (rbk_index* ix : g->parts) member_locks.emplace_back(ix->mu);
  for (rbk_index* ix : g->parts) {
    rbk_status st = tier_check(ix, flags);
    if (st != RBK_OK) return st;
  }
  if (flags == index_flags(g->parts[0])) return RBK_OK;   // the members share their flags
  std::vector<TierPlan> plans(g->G);
  for (int d = 0; d < g->G; ++d) {
    DeviceGuard dg(g->devices[d]);
    rbk_status st = tier_prepare(g->parts[d], flags, &plans[d]);
    if (st != RBK_OK) {
      for (int e = 0; e < d; ++e) {
        DeviceGuard dge(g->devices[e]);
        tier_abort(g->parts[e], &plans[e]);
      }
      return st;
    }
  }
  for (int d = 0; d < g->G; ++d) {
    DeviceGuard dg(g->devices[d]);
    rbk_status st = tier_commit(g->parts[d], &plans[d]);
    if (st != RBK_OK) {   // a CUDA error: release what no member has taken over
      for (int e = d; e < g->G; ++e) {
        DeviceGuard dge(g->devices[e]);
        tier_abort(g->parts[e], &plans[e]);
      }
      return st;
    }
  }
  return RBK_OK;
}

int64_t rbk_group_count(const rbk_group* g) {
  int64_t n = 0;
  if (g)
    for (const rbk_index* ix : g->parts) n += rbk_index_count(ix);
  return n;
}
int64_t rbk_group_size(const rbk_group* g) { return g ? g->n_slots : 0; }
int32_t rbk_group_devices(const rbk_group* g) { return g ? g->G : 0; }
rbk_index* rbk_group_member(rbk_group* g, int32_t i) { return (g && i >= 0 && i < g->G) ? g->parts[i] : nullptr; }
int64_t rbk_group_redone_batches(const rbk_group* g) { return g ? g->redone_batches : 0; }

rbk_status rbk_group_search_f32(rbk_group* g, const float* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                                double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                                float* device_ms_out) {
  return group_search(g, queries, 4, B, query_dim, k_fetch, min_score, out_slots, out_scores, out_counts, device_ms_out);
}
rbk_status rbk_group_search_f64(rbk_group* g, const double* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                                double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                                float* device_ms_out) {
  return group_search(g, queries, 8, B, query_dim, k_fetch, min_score, out_slots, out_scores, out_counts, device_ms_out);
}
rbk_status rbk_group_search_large_f64(rbk_group* g, const double* queries, int32_t B, int32_t query_dim,
                                      int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                      int32_t* out_counts, float* device_ms_out) {
  return group_search_large(g, queries, B, query_dim, k_fetch, min_score, RBK_MAX_K_FETCH_LARGE, out_slots, out_scores,
                            out_counts, device_ms_out);
}
rbk_status rbk_group_search_each_f64(rbk_group* g, const double* queries, int32_t B, int32_t query_dim,
                                     const int32_t* k_fetch, const double* min_score, int64_t* out_slots,
                                     double* out_scores, int32_t* out_counts, float* device_ms_out) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  int K = 0;
  rbk_status st = check_each_args(g->parts[0], B, queries != nullptr, query_dim, k_fetch, min_score, &K);
  if (st != RBK_OK) return st;
  if (B == 0) {
    if (device_ms_out) *device_ms_out = 0.f;
    return RBK_OK;
  }
  // every member runs the route rbk_index_search_each_f64 picks for the batch's largest k
  if (K <= RBK_MAX_K_FETCH)
    return group_search(g, queries, 8, B, query_dim, K, -INFINITY, out_slots, out_scores, out_counts, device_ms_out,
                        k_fetch, min_score);
  return group_search_large(g, queries, B, query_dim, K, -INFINITY, INT32_MAX, out_slots, out_scores, out_counts,
                            device_ms_out, k_fetch, min_score);
}

rbk_status rbk_group_search_slots_f64(rbk_group* g, const int64_t* query_slots, int32_t B, const int32_t* k_fetch,
                                      const double* min_score, int64_t* out_slots, double* out_scores,
                                      int32_t* out_counts, float* device_ms_out) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  int K = 0;
  rbk_status st = check_each_args(g->parts[0], B, query_slots != nullptr, g->dim, k_fetch, min_score, &K);
  if (st != RBK_OK) return st;
  if (device_ms_out) *device_ms_out = 0.f;
  std::lock_guard<std::mutex> lk(g->mu);
  for (int b = 0; b < B; ++b)
    if (query_slots[b] < 0 || query_slots[b] >= g->n_slots)
      return fail(RBK_EINVAL, "query_slots[" + std::to_string(b) + "] is not a slot of this group");
  std::vector<double> q;
  std::vector<int64_t> c_slots;
  std::vector<double> c_scores;
  for (int c0 = 0; c0 < B; c0 += kSlotChunk) {
    const int Bc = std::min(kSlotChunk, B - c0);
    const int Kc = *std::max_element(k_fetch + c0, k_fetch + c0 + Bc);
    q.resize(static_cast<size_t>(Bc) * g->dim);
    st = group_gather(g, query_slots + c0, Bc, q.data());
    if (st != RBK_OK) return st;
    // as in rbk_index_search_slots_f64: a chunk's rows are Kc entries long
    const size_t o = static_cast<size_t>(c0) * K;
    if (Kc < K) {
      c_slots.resize(static_cast<size_t>(Bc) * Kc);
      c_scores.resize(static_cast<size_t>(Bc) * Kc);
    }
    int64_t* cs = Kc < K ? c_slots.data() : out_slots + o;
    double* cd = Kc < K ? c_scores.data() : out_scores + o;
    float ms = 0.f;
    st = Kc <= RBK_MAX_K_FETCH
             ? group_search_locked(g, q.data(), 8, Bc, Kc, -INFINITY, cs, cd, out_counts + c0, &ms, k_fetch + c0,
                                   min_score + c0)
             : group_search_large_locked(g, q.data(), Bc, Kc, -INFINITY, cs, cd, out_counts + c0, &ms, k_fetch + c0,
                                         min_score + c0);
    if (st != RBK_OK) return st;
    if (Kc < K) {
      for (int b = 0; b < Bc; ++b) {
        memcpy(out_slots + o + static_cast<size_t>(b) * K, cs + static_cast<size_t>(b) * Kc, sizeof(int64_t) * Kc);
        memcpy(out_scores + o + static_cast<size_t>(b) * K, cd + static_cast<size_t>(b) * Kc, sizeof(double) * Kc);
      }
      fill_result_tail(out_slots + o, out_scores + o, Bc, K, Kc);
    }
    if (device_ms_out) *device_ms_out += ms;
  }
  return RBK_OK;
}

rbk_status rbk_group_search_mmr_f64(rbk_group* g, const double* queries, int32_t B, int32_t query_dim,
                                    const int32_t* k, const int32_t* fetch_k, const double* lambda_mult,
                                    const double* min_score, int64_t* out_slots, double* out_scores,
                                    int32_t* out_counts, float* device_ms_out) {
  if (!g) return fail(RBK_EINVAL, "null group");
  int K = 0;
  rbk_status st = check_mmr_args(g->parts[0], B, queries != nullptr, query_dim, k, fetch_k, lambda_mult, min_score,
                                 out_slots, out_scores, out_counts, &K);
  if (st != RBK_OK) return st;
  if (device_ms_out) *device_ms_out = 0.f;
  std::lock_guard<std::mutex> lk(g->mu);
  rbk_index* ix0 = g->parts[0];
  // the owners gather the candidates' rows (a candidate is live: a refusal there is a bug) into the pinned g->h_mm in
  // candidate order, from where one asynchronous copy takes them to device_ids[0], which runs the selection; the copy
  // is done before the next query group writes h_mm, since each group ends in a synchronisation of ix0's stream
  MmrStage stage;
  stage.host = [&](const int64_t* slots, int n) -> rbk_status {
    {
      DeviceGuard dg(g->devices[0]);
      CK(g->h_mm.ensure(static_cast<size_t>(n) * g->dim));
    }
    rbk_status s2 = group_gather_locked(g, slots, n, g->h_mm.p, /*allow_dead=*/false);
    if (s2 == RBK_EINVAL) return fail(RBK_ECUDA, std::string("MMR: a candidate row was tombstoned: ") + last_error());
    return s2;
  };
  stage.device = [&](int n) -> rbk_status {
    const size_t bytes = static_cast<size_t>(n) * g->dim * 8;
    CK(ix0->q_raw.ensure(bytes));
    CK(cudaMemcpyAsync(ix0->q_raw.p, g->h_mm.p, bytes, cudaMemcpyHostToDevice, ix0->stream));
    return RBK_OK;
  };
  std::vector<int64_t> c_slots;
  std::vector<double> c_scores;
  std::vector<int32_t> c_counts;
  for (int c0 = 0; c0 < B; c0 += kSlotChunk) {
    const int Bc = std::min(kSlotChunk, B - c0);
    const int F = *std::max_element(fetch_k + c0, fetch_k + c0 + Bc);
    c_slots.resize(static_cast<size_t>(Bc) * F);
    c_scores.resize(static_cast<size_t>(Bc) * F);
    c_counts.resize(Bc);
    const double* q = queries + static_cast<size_t>(c0) * g->dim;
    float ms = 0.f;
    st = F <= RBK_MAX_K_FETCH
             ? group_search_locked(g, q, 8, Bc, F, -INFINITY, c_slots.data(), c_scores.data(), c_counts.data(), &ms,
                                   fetch_k + c0, min_score + c0)
             : group_search_large_locked(g, q, Bc, F, -INFINITY, c_slots.data(), c_scores.data(), c_counts.data(), &ms,
                                         fetch_k + c0, min_score + c0);
    if (st != RBK_OK) return st;
    {
      std::vector<std::unique_lock<std::mutex>> locks;
      for (rbk_index* ix : g->parts) locks.emplace_back(ix->mu);
      DeviceGuard dg(ix0->device);
      const size_t o = static_cast<size_t>(c0) * K;
      st = mmr_select_locked(ix0, Bc, F, c_slots.data(), c_scores.data(), c_counts.data(), k + c0, lambda_mult + c0, K,
                             stage, /*check_dead=*/false, out_slots + o, out_scores + o, out_counts + c0, &ms);
    }
    if (st != RBK_OK) return st;
    if (device_ms_out) *device_ms_out += ms;
  }
  return RBK_OK;
}

rbk_status rbk_group_similar_pairs_f64(rbk_group* g, double min_score, int64_t first_slot, int64_t max_pairs,
                                       int64_t* out_a, int64_t* out_b, double* out_scores, int64_t* n_out,
                                       int64_t* next_slot, float* device_ms_out) {
  if (!g) return fail(RBK_EINVAL, "null group");
  std::lock_guard<std::mutex> lk(g->mu);
  rbk_status st = check_pairs_args(0, g->n_slots, min_score, first_slot, max_pairs, out_a, out_b, out_scores, n_out,
                                   next_slot);
  if (st != RBK_OK) return st;
  std::vector<std::unique_lock<std::mutex>> locks;
  for (rbk_index* ix : g->parts) locks.emplace_back(ix->mu);
  std::vector<int64_t> slots;
  // every member pairs the chunk's rows with its own: the owners gather them into pinned staging, from where one
  // asynchronous copy per member feeds them all at once (the buffer is next written after the chunk's count pass, which
  // every member's stream has finished by then)
  auto load = [&](int64_t a0, int Q) -> rbk_status {
    slots.resize(Q);
    for (int i = 0; i < Q; ++i) slots[i] = a0 + i;
    const size_t n = static_cast<size_t>(Q) * g->dim;
    {
      DeviceGuard dg(g->devices[0]);
      CK(g->h_pq.ensure(n));
    }
    rbk_status s2 = group_gather_locked(g, slots.data(), Q, g->h_pq.p, /*allow_dead=*/true);
    if (s2 != RBK_OK) return s2;
    for (rbk_index* ix : g->parts) {
      DeviceGuard dg(ix->device);
      CK(cudaMemcpyAsync(ix->q_raw.p, g->h_pq.p, sizeof(double) * n, cudaMemcpyHostToDevice, ix->stream));
    }
    return RBK_OK;
  };
  return similar_pairs_run(g->parts, g->n_slots, min_score, first_slot, max_pairs, load, out_a, out_b, out_scores,
                           n_out, next_slot, device_ms_out);
}

rbk_status rbk_group_search_unbounded_f64(rbk_group* g, const double* queries, int32_t B, int32_t query_dim,
                                          int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                          int32_t* out_counts, float* device_ms_out) {
  return group_search_large(g, queries, B, query_dim, k_fetch, min_score, INT32_MAX, out_slots, out_scores, out_counts,
                            device_ms_out);
}

}  // extern "C"
