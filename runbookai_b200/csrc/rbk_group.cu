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
// it and a one-GPU group never needs it.  Exact per-shard fp64 scores make the merge exact; local row order is
// global slot order within a device, so the (score desc, slot asc) tie-break survives (SlotLayout, rbk_internal.h).
#include <dlfcn.h>
#include <nccl.h>   // types and enums only: every NCCL symbol is looked up at run time
#include <string.h>

#include <algorithm>
#include <memory>

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
  std::vector<ncclComm_t> comms; // empty for G == 1
  std::mutex mu;
  struct Dev {
    DevBuf<unsigned char> q, local, all;
  };
  std::vector<Dev> dev;
  DevBuf<unsigned char> out;     // device 0: the merged block (dirty_word)
  PinBuf<unsigned char> h_out, h_q;
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

rbk_status group_append(rbk_group* g, const void* rows, int elem, int64_t n, int64_t* first_out) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (n < 0 || (n > 0 && !rows)) return fail(RBK_EINVAL, "bad rows argument");
  std::lock_guard<std::mutex> lk(g->mu);
  if (first_out) *first_out = g->n_slots;
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

// Stages a batch on every device and enqueues its work there: the buffers for the queries and the packed blocks, the
// start event, the H2D of the queries to each device from one pinned copy (so that the G copies run concurrently, one
// per PCIe link), the member's query scratch, then enqueue(d, ix) with the member's lock held and its device current.
// zero_dirty: the caller reads the dirty count, which the merge kernel adds to - start it from zero (its position
// depends on B and k_fetch, so a running count across calls of different shapes would be garbage).
// q_slack_rows: as for ensure_query_scratch.
template <typename F>
rbk_status stage_and_enqueue(rbk_group* g, const void* queries, int elem, const ResultBlock& L, bool zero_dirty,
                             F&& enqueue, int q_slack_rows = 0) {
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
    if (g->G > 1) CK(g->dev[d].all.ensure(L.bytes * g->G));
    if (d == 0) CK(cudaEventRecord(g->ev0, ix->stream));
    CK(cudaMemcpyAsync(g->dev[d].q.p, g->h_q.p, q_bytes, cudaMemcpyHostToDevice, ix->stream));
    rbk_status st = ensure_query_scratch(ix, B, elem, q_slack_rows);
    if (st != RBK_OK) return st;
    st = enqueue(d, ix);
    if (st != RBK_OK) return st;
  }
  return RBK_OK;
}

// all-gather of the packed blocks (G > 1) + merge on device 0 into g->out; enqueue only
rbk_status exchange_and_merge(rbk_group* g, const ResultBlock& L, int k_fetch) {
  if (g->G > 1) {
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
                         L.flags(o), g->parts[0]->stream));
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

rbk_status group_search(rbk_group* g, const void* queries, int elem, int32_t B, int32_t query_dim, int32_t k_fetch,
                        double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts, float* ms_out) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  rbk_status st = check_search_args(g->parts[0], B, queries != nullptr, query_dim, k_fetch, min_score);
  if (st != RBK_OK) return st;
  if (ms_out) *ms_out = 0.f;
  if (B == 0) return RBK_OK;
  std::lock_guard<std::mutex> lk(g->mu);
  const ResultBlock L(B, k_fetch);
  const int src_type = elem == 8 ? 0 : 1;
  st = stage_and_enqueue(g, queries, elem, L, /*zero_dirty=*/true, [&](int d, rbk_index* ix) {
    unsigned char* l = g->dev[d].local.p;
    return enqueue_search(ix, g->dev[d].q.p, src_type, B, k_fetch, min_score, L.slots(l), L.scores(l), L.counts(l),
                          L.flags(l));
  });
  if (st != RBK_OK) return st;
  st = exchange_and_merge(g, L, k_fetch);
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
      st = rbk_index_search_device(g->parts[d], g->dev[d].q.p, B, k_fetch, min_score, L.slots(l), L.scores(l),
                                   L.counts(l));
      if (st != RBK_OK) return st;
      DeviceGuard dg(g->parts[d]->device);
      CK(cudaMemsetAsync(L.flags(l), 0, static_cast<size_t>(B) * 4, g->parts[d]->stream));   // exact by construction
    }
    st = exchange_and_merge(g, L, k_fetch);
    if (st != RBK_OK) return st;
    st = collect(g, L);
    if (st != RBK_OK) return st;
  }
  if (ms_out) cudaEventElapsedTime(ms_out, g->ev0, g->ev1);
  L.unpack(g->h_out.p, out_slots, out_scores, out_counts);
  return RBK_OK;
}

// Large-k search over the group: count scan + select on every device, ONE wait for all of them (C_q sizes each
// device's candidate buffer), emit scan + exact re-rank on every device into its packed block (flags zero: the
// answers are exact by construction), then the all-gather and merge of group_search.
rbk_status group_search_large(rbk_group* g, const double* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                              double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                              float* ms_out) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  rbk_status st = check_search_args(g->parts[0], B, queries != nullptr, query_dim, k_fetch, min_score,
                                    RBK_MAX_K_FETCH_LARGE);
  if (st != RBK_OK) return st;
  if (ms_out) *ms_out = 0.f;
  if (B == 0) return RBK_OK;
  std::lock_guard<std::mutex> lk(g->mu);
  const ResultBlock L(B, k_fetch);
  st = stage_and_enqueue(g, queries, 8, L, /*zero_dirty=*/false, [&](int d, rbk_index* ix) {
    return large_count(ix, g->dev[d].q.p, B, k_fetch, min_score);
  });
  if (st != RBK_OK) return st;
  for (int d = 0; d < g->G; ++d) {
    DeviceGuard dg(g->parts[d]->device);
    CK(cudaStreamSynchronize(g->parts[d]->stream));
  }
  for (int d = 0; d < g->G; ++d) {
    rbk_index* ix = g->parts[d];
    std::lock_guard<std::mutex> il(ix->mu);
    DeviceGuard dg(ix->device);
    unsigned char* l = g->dev[d].local.p;
    st = large_emit(ix, B, k_fetch, min_score, L.slots(l), L.scores(l), L.counts(l));
    if (st != RBK_OK) return st;
    CK(cudaMemsetAsync(L.flags(l), 0, static_cast<size_t>(B) * 4, ix->stream));
  }
  st = exchange_and_merge(g, L, k_fetch);
  if (st != RBK_OK) return st;
  st = collect(g, L);
  if (st != RBK_OK) return st;
  for (int d = 0; d < g->G; ++d) {   // every device's overflow counter has landed on the host
    if (d > 0) {                     // (collect has waited for device 0)
      DeviceGuard dg(g->parts[d]->device);
      CK(cudaStreamSynchronize(g->parts[d]->stream));
    }
    st = large_check(g->parts[d]);
    if (st != RBK_OK) return st;
  }
  if (ms_out) cudaEventElapsedTime(ms_out, g->ev0, g->ev1);
  L.unpack(g->h_out.p, out_slots, out_scores, out_counts);
  return RBK_OK;
}

// Unbounded search over the group (k_fetch > RBK_MAX_K_FETCH_LARGE; below it, group_search_large): the count scan on
// every device and ONE wait for all of them, then the queries in contiguous groups whose candidates on all devices
// together, plus the result blocks they move, fit kUnboundedBudget.  Per query group: emit scan, exact re-score and
// segmented sort on every device into its packed block of k_eff = count() entries per query, the all-gather and merge
// of group_search, and the copy into the caller's rows of k_fetch entries.
rbk_status group_search_unbounded(rbk_group* g, const double* queries, int32_t B, int32_t query_dim, int32_t k_fetch,
                                  double min_score, int64_t* out_slots, double* out_scores, int32_t* out_counts,
                                  float* ms_out) {
  if (!g) return fail(RBK_EINVAL, "null group");
  if (B > 0 && (!out_slots || !out_scores || !out_counts)) return fail(RBK_EINVAL, "null output");
  rbk_status st = check_search_args(g->parts[0], B, queries != nullptr, query_dim, k_fetch, min_score, INT32_MAX);
  if (st != RBK_OK) return st;
  if (k_fetch <= RBK_MAX_K_FETCH_LARGE)
    return group_search_large(g, queries, B, query_dim, k_fetch, min_score, out_slots, out_scores, out_counts, ms_out);
  if (ms_out) *ms_out = 0.f;
  if (B == 0) return RBK_OK;
  std::lock_guard<std::mutex> lk(g->mu);
  const int k_eff = static_cast<int>(std::min<int64_t>(k_fetch, rbk_group_count(g)));
  fill_result_tail(out_slots, out_scores, B, k_fetch, k_eff);
  if (k_eff == 0) {
    memset(out_counts, 0, sizeof(int32_t) * B);
    return RBK_OK;
  }
  // query groups may start at any query: kBlockM rows of query slack on every member (ensure_query_scratch)
  st = stage_and_enqueue(
      g, queries, 8, ResultBlock(B, 1), /*zero_dirty=*/false,
      [&](int d, rbk_index* ix) { return large_count(ix, g->dev[d].q.p, B, k_eff, min_score); }, kBlockM);
  if (st != RBK_OK) return st;
  for (int d = 0; d < g->G; ++d) {
    DeviceGuard dg(g->parts[d]->device);
    CK(cudaStreamSynchronize(g->parts[d]->stream));
  }
  // a query's cost: its candidates on every device, and its result in the local block, the all-gathered blocks and
  // the merged block
  std::vector<int64_t> cost(B);
  for (int b = 0; b < B; ++b) {
    cost[b] = (g->G + 2) * unbounded_result_bytes(k_eff);
    for (rbk_index* ix : g->parts) cost[b] += ix->h_lcap.p[b] * kUnboundedCandBytes;
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
    if (g->G > 1) CK(g->dev[d].all.ensure(Lmax.bytes * g->G));
    st = unbounded_prepare(ix, B, groups);
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
      st = unbounded_emit(ix, gr.first, gr.second, k_eff, min_score, L.slots(l), L.scores(l), L.counts(l));
      if (st != RBK_OK) return st;
      CK(cudaMemsetAsync(L.flags(l), 0, static_cast<size_t>(Bg) * 4, ix->stream));
    }
    st = exchange_and_merge(g, L, k_eff);
    if (st != RBK_OK) return st;
    st = collect(g, L);
    if (st != RBK_OK) return st;
    unsigned char* h = g->h_out.p;
    for (int b = 0; b < Bg; ++b) {
      const size_t src = static_cast<size_t>(b) * k_eff, dst = static_cast<size_t>(gr.first + b) * k_fetch;
      memcpy(out_slots + dst, L.slots(h) + src, sizeof(int64_t) * k_eff);
      memcpy(out_scores + dst, L.scores(h) + src, sizeof(double) * k_eff);
    }
    memcpy(out_counts + gr.first, L.counts(h), sizeof(int32_t) * Bg);
  }
  for (int d = 0; d < g->G; ++d) {   // every device's overflow counter
    rbk_index* ix = g->parts[d];
    std::lock_guard<std::mutex> il(ix->mu);
    DeviceGuard dg(ix->device);
    st = unbounded_finish(ix);
    if (st != RBK_OK) return st;
    CK(cudaStreamSynchronize(ix->stream));
    st = large_check(ix);
    if (st != RBK_OK) return st;
  }
  if (ms_out) cudaEventElapsedTime(ms_out, g->ev0, g->ev1);
  return RBK_OK;
}

}  // namespace

extern "C" {

rbk_status rbk_group_create(int32_t dim, const int32_t* device_ids, int32_t n_devices, int64_t capacity_hint,
                            uint32_t flags, rbk_group** out) {
  if (!out) return fail(RBK_EINVAL, "out is null");
  *out = nullptr;
  if (!device_ids || n_devices < 1 || n_devices > 64) return fail(RBK_EINVAL, "bad device list");
  for (int a = 0; a < n_devices; ++a)
    for (int b = a + 1; b < n_devices; ++b)
      if (device_ids[a] == device_ids[b]) return fail(RBK_EINVAL, "a device may appear only once in a group");
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
  if (n_devices > 1) {
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
  std::vector<std::vector<int64_t>> local, order;
  split_slots(g, slots, n, &local, &order);
  rbk_status worst = RBK_OK;
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
  return group_search_large(g, queries, B, query_dim, k_fetch, min_score, out_slots, out_scores, out_counts,
                            device_ms_out);
}
rbk_status rbk_group_search_unbounded_f64(rbk_group* g, const double* queries, int32_t B, int32_t query_dim,
                                          int32_t k_fetch, double min_score, int64_t* out_slots, double* out_scores,
                                          int32_t* out_counts, float* device_ms_out) {
  return group_search_unbounded(g, queries, B, query_dim, k_fetch, min_score, out_slots, out_scores, out_counts,
                                device_ms_out);
}

}  // extern "C"
