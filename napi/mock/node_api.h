// node_api.h - MOCK of Node's N-API header, for exercising napi/rbk_napi.cc where Node does not exist.
//
// The build image has neither node nor its headers, so the addon could never be compiled, let alone run.  This
// header declares the ~35 N-API entry points the addon uses with the signatures of Node's own <node_api.h>
// (js_native_api.h / node_api.h, N-API version 6: BigInt64Array is in the typed-array enum), and mock_napi.cc
// implements them over a toy value model (numbers, strings, plain objects, arrays, ArrayBuffers, typed arrays,
// Buffers, classes with wrapped native pointers, promises, async work run on a real second thread).  harness.cc
// plays the part of ts/gpu-embedding-index.ts.  It is test scaffolding: nothing here ships, and passing against
// the mock does not replace a build against real Node - it proves that the addon compiles, links against
// librbk_knn.so, and that its argument handling, error paths and result marshalling do what INTEGRATION.md says.
#ifndef RBK_MOCK_NODE_API_H_
#define RBK_MOCK_NODE_API_H_

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct napi_env__* napi_env;
typedef struct napi_value__* napi_value;
typedef struct napi_ref__* napi_ref;
typedef struct napi_callback_info__* napi_callback_info;
typedef struct napi_deferred__* napi_deferred;
typedef struct napi_async_work__* napi_async_work;

typedef enum {
  napi_ok,
  napi_invalid_arg,
  napi_object_expected,
  napi_string_expected,
  napi_name_expected,
  napi_function_expected,
  napi_number_expected,
  napi_boolean_expected,
  napi_array_expected,
  napi_generic_failure,
  napi_pending_exception,
  napi_cancelled,
  napi_escape_called_twice,
  napi_handle_scope_mismatch,
  napi_callback_scope_mismatch,
  napi_queue_full,
  napi_closing,
  napi_bigint_expected,
  napi_date_expected,
  napi_arraybuffer_expected,
  napi_detachable_arraybuffer_expected,
  napi_would_deadlock
} napi_status;

typedef enum {
  napi_int8_array,
  napi_uint8_array,
  napi_uint8_clamped_array,
  napi_int16_array,
  napi_uint16_array,
  napi_int32_array,
  napi_uint32_array,
  napi_float32_array,
  napi_float64_array,
  napi_bigint64_array,
  napi_biguint64_array
} napi_typedarray_type;

typedef enum {
  napi_default = 0,
  napi_writable = 1 << 0,
  napi_enumerable = 1 << 1,
  napi_configurable = 1 << 2,
  napi_static = 1 << 10
} napi_property_attributes;

typedef napi_value (*napi_callback)(napi_env env, napi_callback_info info);
typedef void (*napi_finalize)(napi_env env, void* finalize_data, void* finalize_hint);
typedef void (*napi_async_execute_callback)(napi_env env, void* data);
typedef void (*napi_async_complete_callback)(napi_env env, napi_status status, void* data);

typedef struct {
  const char* utf8name;
  napi_value name;
  napi_callback method;
  napi_callback getter;
  napi_callback setter;
  napi_value value;
  napi_property_attributes attributes;
  void* data;
} napi_property_descriptor;

#define NAPI_AUTO_LENGTH SIZE_MAX

// -- calls and wrapped objects
napi_status napi_get_cb_info(napi_env env, napi_callback_info cbinfo, size_t* argc, napi_value* argv,
                             napi_value* this_arg, void** data);
napi_status napi_wrap(napi_env env, napi_value js_object, void* native_object, napi_finalize finalize_cb,
                      void* finalize_hint, napi_ref* result);
napi_status napi_unwrap(napi_env env, napi_value js_object, void** result);
napi_status napi_define_class(napi_env env, const char* utf8name, size_t length, napi_callback constructor, void* data,
                              size_t property_count, const napi_property_descriptor* properties, napi_value* result);
// -- reading values
napi_status napi_get_boolean(napi_env env, bool value, napi_value* result);
napi_status napi_get_value_bool(napi_env env, napi_value value, bool* result);
napi_status napi_get_value_string_utf8(napi_env env, napi_value value, char* buf, size_t bufsize, size_t* result);
napi_status napi_has_named_property(napi_env env, napi_value object, const char* utf8name, bool* result);
napi_status napi_get_named_property(napi_env env, napi_value object, const char* utf8name, napi_value* result);
napi_status napi_get_value_int32(napi_env env, napi_value value, int32_t* result);
napi_status napi_get_value_int64(napi_env env, napi_value value, int64_t* result);
napi_status napi_get_value_double(napi_env env, napi_value value, double* result);
napi_status napi_is_array(napi_env env, napi_value value, bool* result);
napi_status napi_get_array_length(napi_env env, napi_value value, uint32_t* result);
napi_status napi_get_element(napi_env env, napi_value object, uint32_t index, napi_value* result);
napi_status napi_get_typedarray_info(napi_env env, napi_value typedarray, napi_typedarray_type* type, size_t* length,
                                     void** data, napi_value* arraybuffer, size_t* byte_offset);
napi_status napi_get_buffer_info(napi_env env, napi_value value, void** data, size_t* length);
// -- creating values
napi_status napi_create_int64(napi_env env, int64_t value, napi_value* result);
napi_status napi_create_string_utf8(napi_env env, const char* str, size_t length, napi_value* result);
napi_status napi_create_error(napi_env env, napi_value code, napi_value msg, napi_value* result);
napi_status napi_create_object(napi_env env, napi_value* result);
napi_status napi_create_arraybuffer(napi_env env, size_t byte_length, void** data, napi_value* result);
napi_status napi_create_typedarray(napi_env env, napi_typedarray_type type, size_t length, napi_value arraybuffer,
                                   size_t byte_offset, napi_value* result);
napi_status napi_set_named_property(napi_env env, napi_value object, const char* utf8name, napi_value value);
// -- exceptions
napi_status napi_throw_error(napi_env env, const char* code, const char* msg);
napi_status napi_throw_type_error(napi_env env, const char* code, const char* msg);
// -- promises and async work
napi_status napi_create_promise(napi_env env, napi_deferred* deferred, napi_value* promise);
napi_status napi_resolve_deferred(napi_env env, napi_deferred deferred, napi_value resolution);
napi_status napi_reject_deferred(napi_env env, napi_deferred deferred, napi_value rejection);
napi_status napi_create_async_work(napi_env env, napi_value async_resource, napi_value async_resource_name,
                                   napi_async_execute_callback execute, napi_async_complete_callback complete,
                                   void* data, napi_async_work* result);
napi_status napi_queue_async_work(napi_env env, napi_async_work work);
napi_status napi_delete_async_work(napi_env env, napi_async_work work);

#ifdef __cplusplus
}
#endif

// Node's NAPI_MODULE registers `regfunc` with the runtime at load time; the mock exports it under a fixed name
// for the harness to call.
#define NAPI_MODULE(modname, regfunc) \
  extern "C" napi_value rbk_mock_module_init(napi_env env, napi_value exports) { return regfunc(env, exports); }

#endif  // RBK_MOCK_NODE_API_H_
