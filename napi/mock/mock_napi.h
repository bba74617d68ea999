// mock_napi.h - what the harness (the "JavaScript side") uses to drive the mock runtime of node_api.h.
#ifndef RBK_MOCK_NAPI_H_
#define RBK_MOCK_NAPI_H_

#include <string>
#include <utility>
#include <vector>

#include "node_api.h"

namespace mock {

napi_env new_env();
void delete_env(napi_env env);   // runs the finalizers of wrapped objects (what GC would do eventually)

// value constructors of the "script"
napi_value undefined(napi_env env);
napi_value number(napi_env env, double v);
napi_value array(napi_env env, const std::vector<napi_value>& elems);
napi_value buffer(napi_env env, const void* bytes, size_t n);                                  // Node Buffer
napi_value typed_array(napi_env env, napi_typedarray_type t, const void* data, size_t length);  // copies the data
napi_value boolean(napi_env env, bool v);
napi_value object(napi_env env, const std::vector<std::pair<std::string, napi_value>>& props);   // { name: value, ... }

// exports.<name>;  new cls(args...);  obj.method(args...).  A thrown exception comes back as false + message.
napi_value get_property(napi_env env, napi_value object, const char* name);
bool construct(napi_env env, napi_value cls, const std::vector<napi_value>& args, napi_value* out, std::string* error);
bool call_method(napi_env env, napi_value object, const char* name, const std::vector<napi_value>& args,
                 napi_value* out, std::string* error);
// obj.name through a getter the class defines
bool get_accessor(napi_env env, napi_value object, const char* name, napi_value* out, std::string* error);

// the event loop: run every queued async work item (execute on a second thread, complete on this one)
void run_event_loop(napi_env env);

// reading results
bool is_undefined(napi_value v);
double as_number(napi_value v);
int as_bool(napi_value v);   // 1 true, 0 false, -1 not a boolean
// promise: 0 pending, 1 fulfilled, 2 rejected; *value = resolution / rejection
int promise_state(napi_value promise, napi_value* value);
std::string error_message(napi_value error);
// typed array contents (pointer into the mock heap, valid until delete_env)
const void* typed_data(napi_value ta, napi_typedarray_type* type, size_t* length);

}  // namespace mock

extern "C" napi_value rbk_mock_module_init(napi_env env, napi_value exports);   // = NAPI_MODULE(..., Init)

#endif
