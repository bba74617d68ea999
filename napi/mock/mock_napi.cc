// mock_napi.cc - a toy implementation of the N-API subset declared in the mock node_api.h (see there).
#include "mock_napi.h"

#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <thread>

namespace {

enum Kind { kUndefined, kBoolean, kNumber, kString, kObject, kArray, kArrayBuffer, kTypedArray, kBuffer, kClass, kPromise, kError };

struct Val {
  Kind kind = kUndefined;
  double num = 0;
  std::string str;                          // string value / error message
  std::map<std::string, Val*> props;        // plain objects, class instances
  std::vector<Val*> elems;                  // arrays
  std::vector<unsigned char> bytes;         // ArrayBuffer / Buffer storage
  // typed array
  napi_typedarray_type ta_type = napi_uint8_array;
  size_t ta_length = 0, ta_offset = 0;
  Val* ta_buffer = nullptr;
  // class
  napi_callback ctor = nullptr;
  std::map<std::string, napi_callback> methods;
  std::map<std::string, napi_callback> getters;
  Val* cls = nullptr;                       // instance -> its class
  // wrapped native pointer
  void* native = nullptr;
  napi_finalize finalize = nullptr;
  void* finalize_hint = nullptr;
  // promise
  int state = 0;
  Val* settled = nullptr;
};

struct Work {
  napi_async_execute_callback execute;
  napi_async_complete_callback complete;
  void* data;
  bool queued = false, deleted = false;
};

struct CallInfo {
  Val* self;
  std::vector<Val*> args;
};

size_t elem_size(napi_typedarray_type t) {
  switch (t) {
    case napi_int8_array: case napi_uint8_array: case napi_uint8_clamped_array: return 1;
    case napi_int16_array: case napi_uint16_array: return 2;
    case napi_int32_array: case napi_uint32_array: case napi_float32_array: return 4;
    default: return 8;
  }
}

}  // namespace

struct napi_env__ {
  std::vector<std::unique_ptr<Val>> heap;
  std::vector<std::unique_ptr<Work>> works;
  std::vector<Work*> queue;
  bool pending = false;
  std::string pending_msg;
  Val* make(Kind k) {
    heap.emplace_back(new Val());
    heap.back()->kind = k;
    return heap.back().get();
  }
};

static inline Val* V(napi_value v) { return reinterpret_cast<Val*>(v); }
static inline napi_value N(Val* v) { return reinterpret_cast<napi_value>(v); }

// ------------------------------------------------------------------------------------------------ N-API subset
extern "C" {

napi_status napi_get_cb_info(napi_env, napi_callback_info cbinfo, size_t* argc, napi_value* argv, napi_value* this_arg,
                             void** data) {
  CallInfo* ci = reinterpret_cast<CallInfo*>(cbinfo);
  if (argc) {
    const size_t room = *argc;
    for (size_t i = 0; i < room && argv; ++i)   // missing arguments read as undefined, as in Node
      argv[i] = i < ci->args.size() ? N(ci->args[i]) : nullptr;
    *argc = ci->args.size();
  }
  if (this_arg) *this_arg = N(ci->self);
  if (data) *data = nullptr;
  return napi_ok;
}

napi_status napi_wrap(napi_env, napi_value js_object, void* native_object, napi_finalize finalize_cb, void* finalize_hint,
                      napi_ref* result) {
  Val* o = V(js_object);
  if (!o || o->kind != kObject) return napi_object_expected;
  if (o->native) return napi_invalid_arg;   // already wrapped
  o->native = native_object;
  o->finalize = finalize_cb;
  o->finalize_hint = finalize_hint;
  if (result) *result = nullptr;
  return napi_ok;
}

napi_status napi_unwrap(napi_env, napi_value js_object, void** result) {
  Val* o = V(js_object);
  if (!o || o->kind != kObject) return napi_object_expected;
  if (!o->native) return napi_invalid_arg;
  *result = o->native;
  return napi_ok;
}

napi_status napi_define_class(napi_env env, const char* utf8name, size_t, napi_callback constructor, void*,
                              size_t property_count, const napi_property_descriptor* properties, napi_value* result) {
  Val* c = env->make(kClass);
  c->str = utf8name;
  c->ctor = constructor;
  for (size_t i = 0; i < property_count; ++i) {
    if (!properties[i].utf8name || (!properties[i].method == !properties[i].getter)) return napi_invalid_arg;
    if (properties[i].method) c->methods[properties[i].utf8name] = properties[i].method;
    else c->getters[properties[i].utf8name] = properties[i].getter;
  }
  *result = N(c);
  return napi_ok;
}

napi_status napi_get_boolean(napi_env env, bool value, napi_value* result) {
  Val* b = env->make(kBoolean);
  b->num = value ? 1 : 0;
  *result = N(b);
  return napi_ok;
}

napi_status napi_get_value_bool(napi_env, napi_value value, bool* result) {
  Val* v = V(value);
  if (!v || v->kind != kBoolean) return napi_boolean_expected;
  *result = v->num != 0;
  return napi_ok;
}

napi_status napi_get_value_string_utf8(napi_env, napi_value value, char* buf, size_t bufsize, size_t* result) {
  Val* v = V(value);
  if (!v || v->kind != kString) return napi_string_expected;
  if (!buf) {
    if (result) *result = v->str.size();
    return napi_ok;
  }
  const size_t n = bufsize == 0 ? 0 : std::min(v->str.size(), bufsize - 1);   // Node truncates and terminates
  if (bufsize) {
    memcpy(buf, v->str.data(), n);
    buf[n] = '\0';
  }
  if (result) *result = n;
  return napi_ok;
}

napi_status napi_has_named_property(napi_env, napi_value object, const char* utf8name, bool* result) {
  Val* o = V(object);
  if (!o || o->kind != kObject) return napi_object_expected;
  *result = o->props.count(utf8name) != 0;
  return napi_ok;
}

napi_status napi_get_named_property(napi_env, napi_value object, const char* utf8name, napi_value* result) {
  Val* o = V(object);
  if (!o || o->kind != kObject) return napi_object_expected;
  auto it = o->props.find(utf8name);
  *result = it == o->props.end() ? nullptr : N(it->second);
  return napi_ok;
}

static napi_status number_of(napi_value value, double* out) {
  Val* v = V(value);
  if (!v || v->kind != kNumber) return napi_number_expected;
  *out = v->num;
  return napi_ok;
}
napi_status napi_get_value_int32(napi_env, napi_value value, int32_t* result) {
  double d;
  napi_status s = number_of(value, &d);
  if (s != napi_ok) return s;
  *result = (d != d || d - d != 0) ? 0 : static_cast<int32_t>(static_cast<int64_t>(d));   // NaN / +-Inf -> 0
  return napi_ok;
}
napi_status napi_get_value_int64(napi_env, napi_value value, int64_t* result) {
  double d;
  napi_status s = number_of(value, &d);
  if (s != napi_ok) return s;
  *result = (d != d || d - d != 0) ? 0 : static_cast<int64_t>(d);
  return napi_ok;
}
napi_status napi_get_value_double(napi_env, napi_value value, double* result) { return number_of(value, result); }

napi_status napi_is_array(napi_env, napi_value value, bool* result) {
  *result = V(value) && V(value)->kind == kArray;
  return napi_ok;
}
napi_status napi_get_array_length(napi_env, napi_value value, uint32_t* result) {
  if (!V(value) || V(value)->kind != kArray) return napi_array_expected;
  *result = static_cast<uint32_t>(V(value)->elems.size());
  return napi_ok;
}
napi_status napi_get_element(napi_env, napi_value object, uint32_t index, napi_value* result) {
  Val* a = V(object);
  if (!a || a->kind != kArray) return napi_object_expected;
  *result = index < a->elems.size() ? N(a->elems[index]) : nullptr;
  return napi_ok;
}
napi_status napi_get_typedarray_info(napi_env, napi_value typedarray, napi_typedarray_type* type, size_t* length,
                                     void** data, napi_value* arraybuffer, size_t* byte_offset) {
  Val* t = V(typedarray);
  if (!t || t->kind != kTypedArray) return napi_invalid_arg;
  if (type) *type = t->ta_type;
  if (length) *length = t->ta_length;
  if (data) *data = t->ta_buffer->bytes.data() + t->ta_offset;
  if (arraybuffer) *arraybuffer = N(t->ta_buffer);
  if (byte_offset) *byte_offset = t->ta_offset;
  return napi_ok;
}
napi_status napi_get_buffer_info(napi_env, napi_value value, void** data, size_t* length) {
  Val* b = V(value);
  if (!b || b->kind != kBuffer) return napi_invalid_arg;
  if (data) *data = b->bytes.data();
  if (length) *length = b->bytes.size();
  return napi_ok;
}

napi_status napi_create_int64(napi_env env, int64_t value, napi_value* result) {
  Val* v = env->make(kNumber);
  v->num = static_cast<double>(value);
  *result = N(v);
  return napi_ok;
}
napi_status napi_create_string_utf8(napi_env env, const char* str, size_t length, napi_value* result) {
  Val* v = env->make(kString);
  v->str = length == NAPI_AUTO_LENGTH ? std::string(str) : std::string(str, length);
  *result = N(v);
  return napi_ok;
}
napi_status napi_create_error(napi_env env, napi_value, napi_value msg, napi_value* result) {
  if (!V(msg) || V(msg)->kind != kString) return napi_string_expected;
  Val* e = env->make(kError);
  e->str = V(msg)->str;
  *result = N(e);
  return napi_ok;
}
napi_status napi_create_object(napi_env env, napi_value* result) {
  *result = N(env->make(kObject));
  return napi_ok;
}
napi_status napi_create_arraybuffer(napi_env env, size_t byte_length, void** data, napi_value* result) {
  Val* b = env->make(kArrayBuffer);
  b->bytes.assign(byte_length, 0);
  if (data) *data = b->bytes.data();
  *result = N(b);
  return napi_ok;
}
napi_status napi_create_typedarray(napi_env env, napi_typedarray_type type, size_t length, napi_value arraybuffer,
                                   size_t byte_offset, napi_value* result) {
  Val* b = V(arraybuffer);
  if (!b || b->kind != kArrayBuffer) return napi_invalid_arg;
  if (byte_offset % elem_size(type) != 0 || byte_offset + length * elem_size(type) > b->bytes.size())
    return napi_invalid_arg;   // Node throws a RangeError here
  Val* t = env->make(kTypedArray);
  t->ta_type = type;
  t->ta_length = length;
  t->ta_offset = byte_offset;
  t->ta_buffer = b;
  *result = N(t);
  return napi_ok;
}
napi_status napi_set_named_property(napi_env, napi_value object, const char* utf8name, napi_value value) {
  Val* o = V(object);
  if (!o || o->kind != kObject) return napi_object_expected;
  o->props[utf8name] = V(value);
  return napi_ok;
}

napi_status napi_throw_error(napi_env env, const char*, const char* msg) {
  env->pending = true;
  env->pending_msg = msg ? msg : "";
  return napi_ok;
}
napi_status napi_throw_type_error(napi_env env, const char* code, const char* msg) {
  return napi_throw_error(env, code, msg);
}

napi_status napi_create_promise(napi_env env, napi_deferred* deferred, napi_value* promise) {
  Val* p = env->make(kPromise);
  *deferred = reinterpret_cast<napi_deferred>(p);
  *promise = N(p);
  return napi_ok;
}
static napi_status settle(napi_deferred deferred, napi_value v, int state) {
  Val* p = reinterpret_cast<Val*>(deferred);
  if (!p || p->kind != kPromise || p->state != 0) return napi_invalid_arg;
  p->state = state;
  p->settled = V(v);
  return napi_ok;
}
napi_status napi_resolve_deferred(napi_env, napi_deferred deferred, napi_value resolution) {
  return settle(deferred, resolution, 1);
}
napi_status napi_reject_deferred(napi_env, napi_deferred deferred, napi_value rejection) {
  return settle(deferred, rejection, 2);
}

napi_status napi_create_async_work(napi_env env, napi_value, napi_value async_resource_name,
                                   napi_async_execute_callback execute, napi_async_complete_callback complete,
                                   void* data, napi_async_work* result) {
  if (!V(async_resource_name) || V(async_resource_name)->kind != kString) return napi_string_expected;
  if (!execute) return napi_invalid_arg;
  env->works.emplace_back(new Work{execute, complete, data});
  *result = reinterpret_cast<napi_async_work>(env->works.back().get());
  return napi_ok;
}
napi_status napi_queue_async_work(napi_env env, napi_async_work work) {
  Work* w = reinterpret_cast<Work*>(work);
  if (!w || w->queued || w->deleted) return napi_invalid_arg;
  w->queued = true;
  env->queue.push_back(w);
  return napi_ok;
}
napi_status napi_delete_async_work(napi_env, napi_async_work work) {
  Work* w = reinterpret_cast<Work*>(work);
  if (!w || w->deleted) return napi_invalid_arg;
  w->deleted = true;
  return napi_ok;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ driver side
namespace mock {

napi_env new_env() { return new napi_env__(); }

void delete_env(napi_env env) {
  for (auto& v : env->heap)
    if (v->kind == kObject && v->native && v->finalize) v->finalize(env, v->native, v->finalize_hint);
  delete env;
}

napi_value undefined(napi_env) { return nullptr; }
napi_value number(napi_env env, double v) {
  Val* n = env->make(kNumber);
  n->num = v;
  return N(n);
}
napi_value array(napi_env env, const std::vector<napi_value>& elems) {
  Val* a = env->make(kArray);
  for (napi_value e : elems) a->elems.push_back(V(e));
  return N(a);
}
napi_value buffer(napi_env env, const void* bytes, size_t n) {
  Val* b = env->make(kBuffer);
  b->bytes.assign(static_cast<const unsigned char*>(bytes), static_cast<const unsigned char*>(bytes) + n);
  return N(b);
}
napi_value typed_array(napi_env env, napi_typedarray_type t, const void* data, size_t length) {
  Val* b = env->make(kArrayBuffer);
  b->bytes.assign(static_cast<const unsigned char*>(data),
                  static_cast<const unsigned char*>(data) + length * elem_size(t));
  Val* ta = env->make(kTypedArray);
  ta->ta_type = t;
  ta->ta_length = length;
  ta->ta_buffer = b;
  return N(ta);
}

napi_value get_property(napi_env, napi_value object, const char* name) {
  Val* o = V(object);
  if (!o) return nullptr;
  auto it = o->props.find(name);
  return it == o->props.end() ? nullptr : N(it->second);
}

static bool invoke(napi_env env, napi_callback cb, Val* self, const std::vector<napi_value>& args, napi_value* out,
                   std::string* error) {
  CallInfo ci;
  ci.self = self;
  for (napi_value a : args) ci.args.push_back(V(a));
  env->pending = false;
  napi_value r = cb(env, reinterpret_cast<napi_callback_info>(&ci));
  if (env->pending) {
    env->pending = false;
    if (error) *error = env->pending_msg;
    return false;
  }
  if (out) *out = r;
  return true;
}

bool construct(napi_env env, napi_value cls, const std::vector<napi_value>& args, napi_value* out, std::string* error) {
  Val* c = V(cls);
  if (!c || c->kind != kClass) {
    if (error) *error = "not a constructor";
    return false;
  }
  Val* self = env->make(kObject);
  self->cls = c;
  napi_value r = nullptr;
  if (!invoke(env, c->ctor, self, args, &r, error)) return false;
  *out = N(self);
  return true;
}

bool call_method(napi_env env, napi_value object, const char* name, const std::vector<napi_value>& args,
                 napi_value* out, std::string* error) {
  Val* o = V(object);
  if (!o || !o->cls || !o->cls->methods.count(name)) {
    if (error) *error = std::string(name) + " is not a function";
    return false;
  }
  return invoke(env, o->cls->methods[name], o, args, out, error);
}

bool get_accessor(napi_env env, napi_value object, const char* name, napi_value* out, std::string* error) {
  Val* o = V(object);
  if (!o || !o->cls || !o->cls->getters.count(name)) {
    if (error) *error = std::string(name) + " is not a getter";
    return false;
  }
  return invoke(env, o->cls->getters[name], o, {}, out, error);
}

napi_value boolean(napi_env env, bool v) {
  napi_value out = nullptr;
  napi_get_boolean(env, v, &out);
  return out;
}

napi_value object(napi_env env, const std::vector<std::pair<std::string, napi_value>>& props) {
  Val* o = env->make(kObject);
  for (const auto& p : props) o->props[p.first] = V(p.second);
  return N(o);
}

int as_bool(napi_value v) { return V(v) && V(v)->kind == kBoolean ? (V(v)->num != 0) : -1; }

void run_event_loop(napi_env env) {
  while (!env->queue.empty()) {
    Work* w = env->queue.front();
    env->queue.erase(env->queue.begin());
    std::thread worker([&] { w->execute(env, w->data); });   // libuv runs `execute` off the JS thread
    worker.join();
    if (w->complete) w->complete(env, napi_ok, w->data);      // ... and `complete` back on it
  }
}

bool is_undefined(napi_value v) { return v == nullptr || V(v)->kind == kUndefined; }
double as_number(napi_value v) { return V(v) && V(v)->kind == kNumber ? V(v)->num : 0.0 / 0.0; }
int promise_state(napi_value promise, napi_value* value) {
  Val* p = V(promise);
  if (!p || p->kind != kPromise) return -1;
  if (value) *value = N(p->settled);
  return p->state;
}
std::string error_message(napi_value error) { return V(error) && V(error)->kind == kError ? V(error)->str : "<not an Error>"; }
const void* typed_data(napi_value ta, napi_typedarray_type* type, size_t* length) {
  Val* t = V(ta);
  if (!t || t->kind != kTypedArray) return nullptr;
  if (type) *type = t->ta_type;
  if (length) *length = t->ta_length;
  return t->ta_buffer->bytes.data() + t->ta_offset;
}

}  // namespace mock
