// harness.cc - plays the JavaScript side of ts/gpu-embedding-index.ts against napi/rbk_napi.cc through the mock
// N-API runtime (mock_napi.cc): loads the module, constructs RbkIndex (one device or a device list, optionally with
// hostRows), loads rows as
// SQLite-style BLOBs and as a Float64Array, overwrites, tombstones, counts, searches through the Promise/async-work
// path, provokes every error path, optionally (compact.txt) tombstones more, compacts and searches again, optionally
// (trim.txt) trims and searches again, clears, and lets the finalizer run.  Inputs and outputs are flat binary files in
// the directory given as argv[1]; tests/test_napi_addon.py writes the inputs and checks the outputs against the
// oracle.  Links against librbk_knn.so (GPU test) or against tests/napi_shim (CPU test).
//
//   harness <dir>        exit 0: scenario ran, results in <dir>;  3: the constructor threw (message in error.txt)
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <fstream>
#include <sstream>

#include "mock_napi.h"

namespace {

std::string g_dir;

template <typename T>
std::vector<T> read_bin(const char* name) {
  std::ifstream f(g_dir + "/" + name, std::ios::binary);
  std::vector<char> raw((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  std::vector<T> out(raw.size() / sizeof(T));
  memcpy(out.data(), raw.data(), out.size() * sizeof(T));
  return out;
}
void write_bin(const char* name, const void* p, size_t bytes) {
  std::ofstream f(g_dir + "/" + name, std::ios::binary);
  f.write(static_cast<const char*>(p), static_cast<std::streamsize>(bytes));
}
void write_text(const char* name, const std::string& s) {
  std::ofstream f(g_dir + "/" + name);
  f << s;
}
[[noreturn]] void die(const std::string& why) {
  fprintf(stderr, "harness: %s\n", why.c_str());
  write_text("error.txt", why);
  exit(2);
}

struct Result {
  std::vector<int64_t> slots;
  std::vector<double> scores;
  std::vector<int32_t> counts;
};

// await ix.search(queries, B, k, minScore): fulfilled -> true + result, rejected -> false + message
bool search(napi_env env, napi_value ix, const std::vector<double>& q, int B, int k, double min_score, Result* r,
            std::string* error, const char* method = "search") {
  napi_value promise = nullptr;
  if (!mock::call_method(env, ix, method,
                         {mock::typed_array(env, napi_float64_array, q.data(), q.size()), mock::number(env, B),
                          mock::number(env, k), mock::number(env, min_score)},
                         &promise, error))
    return false;
  napi_value settled = nullptr;
  if (mock::promise_state(promise, &settled) != 0) die("search() settled its promise before the worker ran");
  mock::run_event_loop(env);
  const int state = mock::promise_state(promise, &settled);
  if (state == 2) {
    *error = mock::error_message(settled);
    return false;
  }
  if (state != 1) die("search() left its promise pending");
  napi_typedarray_type t;
  size_t n;
  const void* p = mock::typed_data(mock::get_property(env, settled, "slots"), &t, &n);
  if (!p || t != napi_bigint64_array || n != static_cast<size_t>(B) * k) die("result.slots is not a BigInt64Array[B*k]");
  r->slots.assign(static_cast<const int64_t*>(p), static_cast<const int64_t*>(p) + n);
  p = mock::typed_data(mock::get_property(env, settled, "scores"), &t, &n);
  if (!p || t != napi_float64_array || n != static_cast<size_t>(B) * k) die("result.scores is not a Float64Array[B*k]");
  r->scores.assign(static_cast<const double*>(p), static_cast<const double*>(p) + n);
  p = mock::typed_data(mock::get_property(env, settled, "counts"), &t, &n);
  if (!p || t != napi_int32_array || n != static_cast<size_t>(B)) die("result.counts is not an Int32Array[B]");
  r->counts.assign(static_cast<const int32_t*>(p), static_cast<const int32_t*>(p) + n);
  return true;
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 2) {
    fprintf(stderr, "usage: harness <dir>\n");
    return 2;
  }
  g_dir = argv[1];
  // meta.txt: dim n_rows n_queries k_fetch min_score n_devices dev0 dev1 ...   (n_devices = 0: a plain ordinal 0)
  int dim = 0, n_rows = 0, n_q = 0, k = 0, n_dev = 0;
  double min_score = 0;
  std::vector<int> devs;
  {
    std::ifstream f(g_dir + "/meta.txt");
    f >> dim >> n_rows >> n_q >> k >> min_score >> n_dev;
    for (int i = 0; i < n_dev; ++i) {
      int d;
      f >> d;
      devs.push_back(d);
    }
    if (!f || dim < 1) die("bad meta.txt");
  }
  const std::vector<double> rows = read_bin<double>("rows.f64");
  const std::vector<double> queries = read_bin<double>("queries.f64");
  const std::vector<int64_t> over_slots = read_bin<int64_t>("over_slots.i64");
  const std::vector<double> over_rows = read_bin<double>("over_rows.f64");
  const std::vector<int64_t> dead = read_bin<int64_t>("dead.i64");
  if (rows.size() != static_cast<size_t>(n_rows) * dim || queries.size() != static_cast<size_t>(n_q) * dim ||
      over_rows.size() != over_slots.size() * dim || over_slots.empty() || dead.empty() || n_rows < 4)
    die("input files do not match meta.txt");

  std::ostringstream log;
  std::string err;
  napi_env env = mock::new_env();
  napi_value exports = nullptr;
  napi_create_object(env, &exports);
  if (rbk_mock_module_init(env, exports) != exports) die("module init did not return exports");
  napi_value cls = mock::get_property(env, exports, "RbkIndex");
  if (!cls) die("exports.RbkIndex is missing");

  // new RbkIndex(dim, device | [devices], capacityHint [, hostRows])
  napi_value dev_arg = mock::number(env, 0);
  if (n_dev > 0) {
    std::vector<napi_value> e;
    for (int d : devs) e.push_back(mock::number(env, d));
    dev_arg = mock::array(env, e);
  }
  // optional host_rows.txt: the constructor's 4th argument (hostRows: float64 rows in pinned host memory)
  std::vector<napi_value> ctor_args = {mock::number(env, dim), dev_arg, mock::number(env, n_rows)};
  {
    std::ifstream hf(g_dir + "/host_rows.txt");
    int host_rows = 0;
    if (hf >> host_rows) ctor_args.push_back(mock::number(env, host_rows));
  }
  napi_value ix = nullptr;
  if (!mock::construct(env, cls, ctor_args, &ix, &err)) {
    write_text("error.txt", err);
    mock::delete_env(env);
    return 3;   // e.g. no CUDA device: the constructor throws, nothing falls back
  }

  // loadBlobs(): the first half as Buffers exactly as better-sqlite3 returns them; then a Float64Array append
  const int half = n_rows / 2;
  napi_value r = nullptr;
  {
    std::vector<napi_value> blobs;
    for (int i = 0; i < half; ++i) blobs.push_back(mock::buffer(env, &rows[static_cast<size_t>(i) * dim], dim * 8));
    if (!mock::call_method(env, ix, "appendBlobs", {mock::array(env, blobs)}, &r, &err)) die("appendBlobs threw: " + err);
    log << "appendBlobs_first " << mock::as_number(r) << "\n";
    if (!mock::call_method(env, ix, "appendF64",
                           {mock::typed_array(env, napi_float64_array, &rows[static_cast<size_t>(half) * dim],
                                              static_cast<size_t>(n_rows - half) * dim)},
                           &r, &err))
      die("appendF64 threw: " + err);
    log << "appendF64_first " << mock::as_number(r) << "\n";
  }
  // set() on existing ids: one through overwriteF64, the rest in one overwriteF64Batch
  if (!mock::call_method(env, ix, "overwriteF64",
                         {mock::number(env, static_cast<double>(over_slots[0])),
                          mock::typed_array(env, napi_float64_array, over_rows.data(), dim)},
                         &r, &err))
    die("overwriteF64 threw: " + err);
  if (!mock::is_undefined(r)) die("overwriteF64 returned a value");
  if (over_slots.size() > 1 &&
      !mock::call_method(env, ix, "overwriteF64Batch",
                         {mock::typed_array(env, napi_bigint64_array, over_slots.data() + 1, over_slots.size() - 1),
                          mock::typed_array(env, napi_float64_array, over_rows.data() + dim,
                                            (over_slots.size() - 1) * dim)},
                         &r, &err))
    die("overwriteF64Batch threw: " + err);
  // deleteMany()
  if (!mock::call_method(env, ix, "tombstone", {mock::typed_array(env, napi_bigint64_array, dead.data(), dead.size())},
                         &r, &err))
    die("tombstone threw: " + err);
  if (!mock::call_method(env, ix, "count", {}, &r, &err)) die("count threw: " + err);
  log << "count " << mock::as_number(r) << "\n";

  // bestBatch()
  Result res;
  if (!search(env, ix, queries, n_q, k, min_score, &res, &err)) die("search rejected: " + err);
  write_bin("slots.i64", res.slots.data(), res.slots.size() * 8);
  write_bin("scores.f64", res.scores.data(), res.scores.size() * 8);
  write_bin("counts.i32", res.counts.data(), res.counts.size() * 4);

  // searchLarge(): optional large.txt lists k_fetch values (up to 4096); results land in large<i>_*.  One more call
  // with k_fetch 4097 must reject with the library's message.
  {
    std::ifstream lf(g_dir + "/large.txt");
    int kl, i = 0;
    bool any = false;
    while (lf >> kl) {
      any = true;
      Result lr;
      if (!search(env, ix, queries, n_q, kl, min_score, &lr, &err, "searchLarge")) die("searchLarge rejected: " + err);
      const std::string p = "large" + std::to_string(i++) + "_";
      write_bin((p + "slots.i64").c_str(), lr.slots.data(), lr.slots.size() * 8);
      write_bin((p + "scores.f64").c_str(), lr.scores.data(), lr.scores.size() * 8);
      write_bin((p + "counts.i32").c_str(), lr.counts.data(), lr.counts.size() * 4);
    }
    if (any) {
      Result none;
      if (search(env, ix, queries, n_q, 4097, min_score, &none, &err, "searchLarge"))
        die("searchLarge with k_fetch 4097 did not reject");
      log << "err_large " << err << "\n";
    }
  }

  // searchUnbounded(): optional unbounded.txt lists k_fetch values (any >= 1); results land in unbounded<i>_*.  One
  // more call with k_fetch 0 must reject with the library's message.
  {
    std::ifstream uf(g_dir + "/unbounded.txt");
    int ku, i = 0;
    bool any = false;
    while (uf >> ku) {
      any = true;
      Result ur;
      if (!search(env, ix, queries, n_q, ku, min_score, &ur, &err, "searchUnbounded"))
        die("searchUnbounded rejected: " + err);
      const std::string p = "unbounded" + std::to_string(i++) + "_";
      write_bin((p + "slots.i64").c_str(), ur.slots.data(), ur.slots.size() * 8);
      write_bin((p + "scores.f64").c_str(), ur.scores.data(), ur.scores.size() * 8);
      write_bin((p + "counts.i32").c_str(), ur.counts.data(), ur.counts.size() * 4);
    }
    if (any) {
      Result none;
      if (search(env, ix, queries, n_q, 0, min_score, &none, &err, "searchUnbounded"))
        die("searchUnbounded with k_fetch 0 did not reject");
      log << "err_unbounded " << err << "\n";
    }
  }

  // ---- error paths: each must surface as a JS exception / rejection with the reference's wording
  {
    std::vector<double> odd(static_cast<size_t>(dim) + 1, 1.0);
    if (mock::call_method(env, ix, "appendF64", {mock::typed_array(env, napi_float64_array, odd.data(), odd.size())}, &r,
                          &err))
      die("appendF64 of a wrong-length vector did not throw");
    log << "err_append " << err << "\n";
    std::vector<double> oddq(static_cast<size_t>(n_q) * (dim + 1), 1.0);
    Result none;
    if (search(env, ix, oddq, n_q, k, min_score, &none, &err)) die("search with wrong-length queries did not reject");
    log << "err_search " << err << "\n";
    if (mock::call_method(env, ix, "tombstone", {mock::typed_array(env, napi_float64_array, odd.data(), 1)}, &r, &err))
      die("tombstone(Float64Array) did not throw");
    log << "err_tombstone " << err << "\n";
    if (mock::call_method(env, ix, "overwriteF64Batch",
                          {mock::typed_array(env, napi_bigint64_array, dead.data(), 1),
                           mock::typed_array(env, napi_float64_array, over_rows.data(), dim)},
                          &r, &err))
      die("overwriteF64Batch of a tombstoned slot did not throw");
    log << "err_overwrite_dead " << err << "\n";
    if (mock::call_method(env, ix, "overwriteF64Batch",
                          {mock::typed_array(env, napi_bigint64_array, dead.data(), 1),
                           mock::typed_array(env, napi_float64_array, over_rows.data(), dim - 1 > 0 ? dim - 1 : 1)},
                          &r, &err) && dim > 1)
      die("overwriteF64Batch with a short row did not throw");
    log << "err_overwrite_len " << err << "\n";
    // the same search again: errors above must not have disturbed the index
    Result again;
    if (!search(env, ix, queries, n_q, k, min_score, &again, &err)) die("second search rejected: " + err);
    log << "repeat_identical "
        << (again.slots == res.slots && again.counts == res.counts &&
            memcmp(again.scores.data(), res.scores.data(), res.scores.size() * 8) == 0)
        << "\n";
  }

  Result latest = res;   // the answer of the index as it stands
  // compact(): optional compact.txt lists more slots to tombstone first; then compact() and the same search again,
  // results in compact_*.  On a device-group handle compact() must throw (logged as err_compact).
  {
    std::ifstream cf(g_dir + "/compact.txt");
    std::vector<int64_t> more;
    int64_t s;
    while (cf >> s) more.push_back(s);
    if (!more.empty()) {
      if (!mock::call_method(env, ix, "tombstone",
                             {mock::typed_array(env, napi_bigint64_array, more.data(), more.size())}, &r, &err))
        die("tombstone before compact threw: " + err);
      if (!mock::call_method(env, ix, "compact", {}, &r, &err)) {
        if (n_dev == 0) die("compact threw: " + err);
        log << "err_compact " << err << "\n";
      } else {
        napi_typedarray_type t;
        size_t n;
        const void* p = mock::typed_data(r, &t, &n);
        if (!p || t != napi_bigint64_array || n != static_cast<size_t>(n_rows)) die("compact() is not a BigInt64Array[n_rows]");
        write_bin("compact_map.i64", p, n * 8);
        if (!mock::call_method(env, ix, "count", {}, &r, &err)) die("count threw: " + err);
        log << "count_after_compact " << mock::as_number(r) << "\n";
        Result cr;
        if (!search(env, ix, queries, n_q, k, min_score, &cr, &err)) die("search after compact rejected: " + err);
        write_bin("compact_slots.i64", cr.slots.data(), cr.slots.size() * 8);
        write_bin("compact_scores.f64", cr.scores.data(), cr.scores.size() * 8);
        write_bin("compact_counts.i32", cr.counts.data(), cr.counts.size() * 4);
        latest = cr;
      }
    }
  }

  // trim(): optional trim.txt; trim() and the same search again, results in trim_*, which must equal the answer before
  // the trim (logged as trim_identical).
  {
    std::ifstream tf(g_dir + "/trim.txt");
    if (tf.good()) {
      if (!mock::call_method(env, ix, "trim", {}, &r, &err)) die("trim threw: " + err);
      if (!mock::is_undefined(r)) die("trim returned a value");
      Result tr;
      if (!search(env, ix, queries, n_q, k, min_score, &tr, &err)) die("search after trim rejected: " + err);
      write_bin("trim_slots.i64", tr.slots.data(), tr.slots.size() * 8);
      write_bin("trim_scores.f64", tr.scores.data(), tr.scores.size() * 8);
      write_bin("trim_counts.i32", tr.counts.data(), tr.counts.size() * 4);
      log << "trim_identical "
          << (tr.slots == latest.slots && tr.counts == latest.counts &&
              memcmp(tr.scores.data(), latest.scores.data(), latest.scores.size() * 8) == 0)
          << "\n";
    }
  }

  // clear(): Map.clear
  if (!mock::call_method(env, ix, "clear", {}, &r, &err)) die("clear threw: " + err);
  if (!mock::call_method(env, ix, "count", {}, &r, &err)) die("count threw: " + err);
  log << "count_after_clear " << mock::as_number(r) << "\n";
  Result empty;
  if (!search(env, ix, queries, n_q, k, min_score, &empty, &err)) die("search after clear rejected: " + err);
  int hits = 0;
  for (int32_t c : empty.counts) hits += c;
  log << "hits_after_clear " << hits << "\n";

  mock::delete_env(env);   // "GC": finalize_index destroys the native handle
  log << "finalized 1\n";
  write_text("log.txt", log.str());
  return 0;
}
