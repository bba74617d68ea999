// harness.cc - plays the JavaScript side of ts/gpu-embedding-index.ts against napi/rbk_napi.cc through the mock
// N-API runtime (mock_napi.cc): loads the module, constructs RbkIndex (one device or a device list, optionally with
// hostRows), loads rows as
// SQLite-style BLOBs and as a Float64Array, overwrites, tombstones, counts, searches through the Promise/async-work
// path, provokes every error path, optionally (compact.txt) tombstones more, compacts and searches again, optionally
// (trim.txt) trims and searches again, optionally (set_tier.txt) changes the storage tier between searches, clears, and
// lets the finalizer run.  Inputs and outputs are flat binary files in
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
  // optional host_rows.txt: the constructor's 4th argument (hostRows: float64 rows in pinned host memory);
  // optional scan_f16.txt: its 5th (scanF16: the scan reads fp16 rows), with hostRows 0 unless host_rows.txt says
  std::vector<napi_value> ctor_args = {mock::number(env, dim), dev_arg, mock::number(env, n_rows)};
  {
    std::ifstream hf(g_dir + "/host_rows.txt"), sf(g_dir + "/scan_f16.txt");
    int host_rows = 0, scan_f16 = 0;
    const bool have_host = static_cast<bool>(hf >> host_rows);
    const bool have_f16 = static_cast<bool>(sf >> scan_f16);
    if (have_host || have_f16) ctor_args.push_back(mock::number(env, host_rows));
    if (have_f16) ctor_args.push_back(mock::number(env, scan_f16));
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

  // setTier() / tier: optional set_tier.txt "f64OnHost scanF16" (0 or 1 each).  Reads `tier`, changes both, searches
  // again (results in tier_*, logged as tier_identical), flips scanF16 alone and searches again (tier_partial_identical),
  // then passes a number where a boolean belongs (err_set_tier_type).  A library without tier changes: err_set_tier.
  {
    std::ifstream sf(g_dir + "/set_tier.txt");
    int host = 0, f16 = 0;
    if (sf >> host >> f16) {
      napi_value t = nullptr;
      auto log_tier = [&](const char* key) {
        if (!mock::get_accessor(env, ix, "tier", &t, &err)) return false;
        log << key << " " << mock::as_bool(mock::get_property(env, t, "f64OnHost")) << " "
            << mock::as_bool(mock::get_property(env, t, "scanF16")) << "\n";
        return true;
      };
      auto same_as_first = [&](const Result& x) {
        return x.slots == res.slots && x.counts == res.counts &&
               memcmp(x.scores.data(), res.scores.data(), res.scores.size() * 8) == 0;
      };
      if (!log_tier("tier_before")) {
        log << "err_set_tier " << err << "\n";
      } else {
        napi_value arg = mock::object(env, {{"f64OnHost", mock::boolean(env, host != 0)},
                                            {"scanF16", mock::boolean(env, f16 != 0)}});
        if (!mock::call_method(env, ix, "setTier", {arg}, &r, &err)) die("setTier threw: " + err);
        if (!mock::is_undefined(r)) die("setTier returned a value");
        log_tier("tier_after");
        Result tr;
        if (!search(env, ix, queries, n_q, k, min_score, &tr, &err)) die("search after setTier rejected: " + err);
        write_bin("tier_slots.i64", tr.slots.data(), tr.slots.size() * 8);
        write_bin("tier_scores.f64", tr.scores.data(), tr.scores.size() * 8);
        write_bin("tier_counts.i32", tr.counts.data(), tr.counts.size() * 4);
        log << "tier_identical " << same_as_first(tr) << "\n";
        if (!mock::call_method(env, ix, "setTier", {mock::object(env, {{"scanF16", mock::boolean(env, f16 == 0)}})}, &r,
                               &err))
          die("setTier({scanF16}) threw: " + err);
        log_tier("tier_partial");
        Result pr;
        if (!search(env, ix, queries, n_q, k, min_score, &pr, &err)) die("search after setTier rejected: " + err);
        log << "tier_partial_identical " << same_as_first(pr) << "\n";
        if (mock::call_method(env, ix, "setTier", {mock::object(env, {{"f64OnHost", mock::number(env, 1)}})}, &r, &err))
          die("setTier with a number did not throw");
        log << "err_set_tier_type " << err << "\n";
      }
    }
  }

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

  // searchEach(): optional each.txt holds one "kFetch minScore" pair per query (minScore may be -inf); results land in
  // each_* with rows of K = max kFetch entries.  has_search_each.txt gets the hasSearchEach getter first.  Then one call
  // with a kFetch of 0 must reject with the library's message (err_each), and one with a short kFetch must throw
  // (err_each_len).
  {
    std::ifstream ef(g_dir + "/each.txt");
    std::vector<int32_t> ke;
    std::vector<double> me;
    std::string ks, ms;
    while (ef >> ks >> ms) {
      ke.push_back(static_cast<int32_t>(strtol(ks.c_str(), nullptr, 10)));
      me.push_back(strtod(ms.c_str(), nullptr));
    }
    if (!ke.empty()) {
      if (ke.size() != static_cast<size_t>(n_q)) die("each.txt needs one pair per query");
      napi_value has = nullptr;
      if (!mock::get_accessor(env, ix, "hasSearchEach", &has, &err)) die("hasSearchEach threw: " + err);
      write_text("has_search_each.txt", mock::as_bool(has) ? "1" : "0");
      int K = 0;
      for (int32_t v : ke) K = v > K ? v : K;
      auto call_each = [&](const std::vector<int32_t>& kv, Result* out) {
        napi_value promise = nullptr, settled = nullptr;
        if (!mock::call_method(env, ix, "searchEach",
                               {mock::typed_array(env, napi_float64_array, queries.data(), queries.size()),
                                mock::number(env, n_q), mock::typed_array(env, napi_int32_array, kv.data(), kv.size()),
                                mock::typed_array(env, napi_float64_array, me.data(), me.size())},
                               &promise, &err))
          return false;
        mock::run_event_loop(env);
        const int state = mock::promise_state(promise, &settled);
        if (state == 2) {
          err = mock::error_message(settled);
          return false;
        }
        if (state != 1) die("searchEach() left its promise pending");
        napi_typedarray_type t;
        size_t n;
        const void* p = mock::typed_data(mock::get_property(env, settled, "slots"), &t, &n);
        if (!p || t != napi_bigint64_array || n != static_cast<size_t>(n_q) * K) die("searchEach slots are not [B*K]");
        out->slots.assign(static_cast<const int64_t*>(p), static_cast<const int64_t*>(p) + n);
        p = mock::typed_data(mock::get_property(env, settled, "scores"), &t, &n);
        if (!p || t != napi_float64_array || n != static_cast<size_t>(n_q) * K) die("searchEach scores are not [B*K]");
        out->scores.assign(static_cast<const double*>(p), static_cast<const double*>(p) + n);
        p = mock::typed_data(mock::get_property(env, settled, "counts"), &t, &n);
        if (!p || t != napi_int32_array || n != static_cast<size_t>(n_q)) die("searchEach counts are not [B]");
        out->counts.assign(static_cast<const int32_t*>(p), static_cast<const int32_t*>(p) + n);
        return true;
      };
      Result er;
      if (!call_each(ke, &er)) die("searchEach rejected: " + err);
      write_bin("each_slots.i64", er.slots.data(), er.slots.size() * 8);
      write_bin("each_scores.f64", er.scores.data(), er.scores.size() * 8);
      write_bin("each_counts.i32", er.counts.data(), er.counts.size() * 4);
      std::vector<int32_t> bad = ke;
      bad[0] = 0;
      Result none;
      if (call_each(bad, &none)) die("searchEach with a kFetch of 0 did not reject");
      log << "err_each " << err << "\n";
      bad.pop_back();
      if (call_each(bad, &none)) die("searchEach with a short kFetch did not throw");
      log << "err_each_len " << err << "\n";
    }
  }

  // searchSlots(): optional slots.txt holds "slot kFetch minScore" triples (minScore may be -inf); results land in
  // slots_* with rows of K = max kFetch entries.  has_search_slots.txt gets the hasSearchSlots getter first.  Then one
  // call with a kFetch of 0 must reject with the library's message (err_slots), and one naming a slot past the end
  // too (err_slots_range).
  {
    std::ifstream sf(g_dir + "/slots.txt");
    std::vector<int64_t> qs;
    std::vector<int32_t> ks_v;
    std::vector<double> ms_v;
    std::string ss, ks, ms;
    while (sf >> ss >> ks >> ms) {
      qs.push_back(strtoll(ss.c_str(), nullptr, 10));
      ks_v.push_back(static_cast<int32_t>(strtol(ks.c_str(), nullptr, 10)));
      ms_v.push_back(strtod(ms.c_str(), nullptr));
    }
    if (!qs.empty()) {
      napi_value has = nullptr;
      if (!mock::get_accessor(env, ix, "hasSearchSlots", &has, &err)) die("hasSearchSlots threw: " + err);
      write_text("has_search_slots.txt", mock::as_bool(has) ? "1" : "0");
      const int nb = static_cast<int>(qs.size());
      int K = 0;
      for (int32_t v : ks_v) K = v > K ? v : K;
      auto call_slots = [&](const std::vector<int64_t>& sv, const std::vector<int32_t>& kv, Result* out) {
        napi_value promise = nullptr, settled = nullptr;
        if (!mock::call_method(env, ix, "searchSlots",
                               {mock::typed_array(env, napi_bigint64_array, sv.data(), sv.size()), mock::number(env, nb),
                                mock::typed_array(env, napi_int32_array, kv.data(), kv.size()),
                                mock::typed_array(env, napi_float64_array, ms_v.data(), ms_v.size())},
                               &promise, &err))
          return false;
        mock::run_event_loop(env);
        const int state = mock::promise_state(promise, &settled);
        if (state == 2) {
          err = mock::error_message(settled);
          return false;
        }
        if (state != 1) die("searchSlots() left its promise pending");
        napi_typedarray_type t;
        size_t n;
        const void* p = mock::typed_data(mock::get_property(env, settled, "slots"), &t, &n);
        if (!p || t != napi_bigint64_array || n != static_cast<size_t>(nb) * K) die("searchSlots slots are not [B*K]");
        out->slots.assign(static_cast<const int64_t*>(p), static_cast<const int64_t*>(p) + n);
        p = mock::typed_data(mock::get_property(env, settled, "scores"), &t, &n);
        if (!p || t != napi_float64_array || n != static_cast<size_t>(nb) * K) die("searchSlots scores are not [B*K]");
        out->scores.assign(static_cast<const double*>(p), static_cast<const double*>(p) + n);
        p = mock::typed_data(mock::get_property(env, settled, "counts"), &t, &n);
        if (!p || t != napi_int32_array || n != static_cast<size_t>(nb)) die("searchSlots counts are not [B]");
        out->counts.assign(static_cast<const int32_t*>(p), static_cast<const int32_t*>(p) + n);
        return true;
      };
      Result sr;
      if (!call_slots(qs, ks_v, &sr)) die("searchSlots rejected: " + err);
      write_bin("slots_slots.i64", sr.slots.data(), sr.slots.size() * 8);
      write_bin("slots_scores.f64", sr.scores.data(), sr.scores.size() * 8);
      write_bin("slots_counts.i32", sr.counts.data(), sr.counts.size() * 4);
      std::vector<int32_t> bad = ks_v;
      bad[0] = 0;
      Result none;
      if (call_slots(qs, bad, &none)) die("searchSlots with a kFetch of 0 did not reject");
      log << "err_slots " << err << "\n";
      std::vector<int64_t> far = qs;
      far[0] = int64_t{1} << 40;
      if (call_slots(far, ks_v, &none)) die("searchSlots past the last slot did not reject");
      log << "err_slots_range " << err << "\n";
    }
  }

  // similarPairs(): optional pairs.txt holds "minScore maxPairs" (minScore may be -inf).  has_similar_pairs.txt gets the
  // hasSimilarPairs getter first; then the pages from slot 0 on, each of at most maxPairs entries, until nextSlot is
  // n_rows, land concatenated in pairs_a / pairs_b / pairs_scores, and the page count in pairs_pages.txt.  Then one call
  // with maxPairs 0 must reject with the library's message (err_pairs).
  {
    std::ifstream pf(g_dir + "/pairs.txt");
    std::string ms_s, mp_s;
    if (pf >> ms_s >> mp_s) {
      napi_value has = nullptr;
      if (!mock::get_accessor(env, ix, "hasSimilarPairs", &has, &err)) die("hasSimilarPairs threw: " + err);
      write_text("has_similar_pairs.txt", mock::as_bool(has) ? "1" : "0");
      const double ms = strtod(ms_s.c_str(), nullptr);
      const double mp = strtod(mp_s.c_str(), nullptr);
      std::vector<int64_t> all_a, all_b;
      std::vector<double> all_s;
      auto call_pairs = [&](double first, double max_pairs, double* next) {
        napi_value promise = nullptr, settled = nullptr;
        if (!mock::call_method(env, ix, "similarPairs",
                               {mock::number(env, ms), mock::number(env, first), mock::number(env, max_pairs)},
                               &promise, &err))
          return false;
        mock::run_event_loop(env);
        const int state = mock::promise_state(promise, &settled);
        if (state == 2) {
          err = mock::error_message(settled);
          return false;
        }
        if (state != 1) die("similarPairs() left its promise pending");
        napi_typedarray_type t;
        size_t na, nb, nv;
        const void* pa = mock::typed_data(mock::get_property(env, settled, "a"), &t, &na);
        if (!pa || t != napi_bigint64_array) die("similarPairs a is not a BigInt64Array");
        const void* pb = mock::typed_data(mock::get_property(env, settled, "b"), &t, &nb);
        if (!pb || t != napi_bigint64_array) die("similarPairs b is not a BigInt64Array");
        const void* pv = mock::typed_data(mock::get_property(env, settled, "scores"), &t, &nv);
        if (!pv || t != napi_float64_array) die("similarPairs scores is not a Float64Array");
        if (na != nb || na != nv || na > static_cast<size_t>(max_pairs)) die("similarPairs arrays disagree");
        all_a.insert(all_a.end(), static_cast<const int64_t*>(pa), static_cast<const int64_t*>(pa) + na);
        all_b.insert(all_b.end(), static_cast<const int64_t*>(pb), static_cast<const int64_t*>(pb) + nb);
        all_s.insert(all_s.end(), static_cast<const double*>(pv), static_cast<const double*>(pv) + nv);
        *next = mock::as_number(mock::get_property(env, settled, "nextSlot"));
        return true;
      };
      double next = 0;
      int pages = 0;
      while (next < n_rows) {
        double after = 0;
        if (!call_pairs(next, mp, &after)) die("similarPairs rejected: " + err);
        if (!(after > next)) die("similarPairs made no progress");
        next = after;
        ++pages;
      }
      write_bin("pairs_a.i64", all_a.data(), all_a.size() * 8);
      write_bin("pairs_b.i64", all_b.data(), all_b.size() * 8);
      write_bin("pairs_scores.f64", all_s.data(), all_s.size() * 8);
      write_text("pairs_pages.txt", std::to_string(pages));
      double none = 0;
      if (call_pairs(0, 0, &none)) die("similarPairs with maxPairs 0 did not reject");
      log << "err_pairs " << err << "\n";
    }
  }

  // searchMmr(): optional mmr.txt holds one "k fetchK lambdaMult minScore" line per query (minScore may be -inf);
  // results land in mmr_* with rows of K = max k entries.  has_search_mmr.txt gets the hasSearchMmr getter first.  Then
  // one call with a k of 0 (err_mmr) and one with a lambdaMult of 2 (err_mmr_lambda) must reject with the library's
  // message.
  {
    std::ifstream mf(g_dir + "/mmr.txt");
    std::vector<int32_t> kv, fv;
    std::vector<double> lv, mv;
    std::string ks, fs, ls, ms;
    while (mf >> ks >> fs >> ls >> ms) {
      kv.push_back(static_cast<int32_t>(strtol(ks.c_str(), nullptr, 10)));
      fv.push_back(static_cast<int32_t>(strtol(fs.c_str(), nullptr, 10)));
      lv.push_back(strtod(ls.c_str(), nullptr));
      mv.push_back(strtod(ms.c_str(), nullptr));
    }
    if (!kv.empty()) {
      if (kv.size() != static_cast<size_t>(n_q)) die("mmr.txt needs one line per query");
      napi_value has = nullptr;
      if (!mock::get_accessor(env, ix, "hasSearchMmr", &has, &err)) die("hasSearchMmr threw: " + err);
      write_text("has_search_mmr.txt", mock::as_bool(has) ? "1" : "0");
      int K = 0;
      for (int32_t v : kv) K = v > K ? v : K;
      auto call_mmr = [&](const std::vector<int32_t>& k, const std::vector<double>& lam, Result* out) {
        napi_value promise = nullptr, settled = nullptr;
        if (!mock::call_method(env, ix, "searchMmr",
                               {mock::typed_array(env, napi_float64_array, queries.data(), queries.size()),
                                mock::number(env, n_q), mock::typed_array(env, napi_int32_array, k.data(), k.size()),
                                mock::typed_array(env, napi_int32_array, fv.data(), fv.size()),
                                mock::typed_array(env, napi_float64_array, lam.data(), lam.size()),
                                mock::typed_array(env, napi_float64_array, mv.data(), mv.size())},
                               &promise, &err))
          return false;
        mock::run_event_loop(env);
        const int state = mock::promise_state(promise, &settled);
        if (state == 2) {
          err = mock::error_message(settled);
          return false;
        }
        if (state != 1) die("searchMmr() left its promise pending");
        napi_typedarray_type t;
        size_t n;
        const void* p = mock::typed_data(mock::get_property(env, settled, "slots"), &t, &n);
        if (!p || t != napi_bigint64_array || n != static_cast<size_t>(n_q) * K) die("searchMmr slots are not [B*K]");
        out->slots.assign(static_cast<const int64_t*>(p), static_cast<const int64_t*>(p) + n);
        p = mock::typed_data(mock::get_property(env, settled, "scores"), &t, &n);
        if (!p || t != napi_float64_array || n != static_cast<size_t>(n_q) * K) die("searchMmr scores are not [B*K]");
        out->scores.assign(static_cast<const double*>(p), static_cast<const double*>(p) + n);
        p = mock::typed_data(mock::get_property(env, settled, "counts"), &t, &n);
        if (!p || t != napi_int32_array || n != static_cast<size_t>(n_q)) die("searchMmr counts are not [B]");
        out->counts.assign(static_cast<const int32_t*>(p), static_cast<const int32_t*>(p) + n);
        return true;
      };
      Result mr;
      if (!call_mmr(kv, lv, &mr)) die("searchMmr rejected: " + err);
      write_bin("mmr_slots.i64", mr.slots.data(), mr.slots.size() * 8);
      write_bin("mmr_scores.f64", mr.scores.data(), mr.scores.size() * 8);
      write_bin("mmr_counts.i32", mr.counts.data(), mr.counts.size() * 4);
      Result none;
      std::vector<int32_t> bad_k = kv;
      bad_k[0] = 0;
      if (call_mmr(bad_k, lv, &none)) die("searchMmr with a k of 0 did not reject");
      log << "err_mmr " << err << "\n";
      std::vector<double> bad_l = lv;
      bad_l[0] = 2.0;
      if (call_mmr(kv, bad_l, &none)) die("searchMmr with a lambdaMult of 2 did not reject");
      log << "err_mmr_lambda " << err << "\n";
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
