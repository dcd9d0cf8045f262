// napi_mock.cc -- TEST INFRASTRUCTURE: a miniature in-process implementation of the N-API
// subset declared in tests/stubs/node_api.h, so that js/src/binding.cc (the addon a manatee
// maintainer builds against Node) can be compiled, linked and EXECUTED here without Node:
//   * on the CPU, against tests/stubs/mtz_mock.cc (an in-memory stand-in for the library),
//     to check the binding's own logic: argument marshalling, error throwing, the
//     eventfd -> poll thread -> threadsafe-function wake-up path, external ArrayBuffers;
//   * on an H100, against the real libmanatee_gpu.so: the same exported functions the JS
//     Transform calls, driven in the same order, moving a real stream through the GPU.
// What it does not cover is V8 itself and js/lib/gpuSnapshotStage.js.
#include "node_api.h"
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <deque>
#include <map>
#include <mutex>
#include <string>
#include <vector>
#include "napi_mock.h"

struct napi_env__ {
	bool pending = false;
	std::string code, msg;
	std::vector<napi_value> pool;          // everything allocated, freed at exit
	std::mutex mu;
	std::condition_variable cv;
	std::deque<napi_threadsafe_function> ready;    // the "event loop" queue
};

struct napi_callback_info__ { std::vector<napi_value> argv; };

struct napi_threadsafe_function__ {
	napi_env env;
	napi_value fn;
	bool released = false;
};

static napi_value mk(napi_env env, mock_kind k)
{
	napi_value v = new napi_value__();
	v->kind = k;
	std::lock_guard<std::mutex> g(env->mu);
	env->pool.push_back(v);
	return v;
}

// ---------------------------------------------------------------- harness side
napi_env mock_env_new() { return new napi_env__(); }
bool mock_exception(napi_env env, std::string *code, std::string *msg)
{
	if (!env->pending) return false;
	if (code) *code = env->code;
	if (msg) *msg = env->msg;
	env->pending = false;
	return true;
}
napi_value mock_number(napi_env env, double d) { napi_value v = mk(env, MK_NUMBER); v->num = d; return v; }
napi_value mock_object(napi_env env) { return mk(env, MK_OBJECT); }
napi_value mock_buffer(napi_env env, void *p, size_t n) { napi_value v = mk(env, MK_BUFFER); v->ptr = p; v->len = n; return v; }
napi_value mock_function(napi_env env, std::function<void()> f) { napi_value v = mk(env, MK_FUNCTION); v->fn = f; return v; }
void mock_set(napi_value obj, const char *name, napi_value v) { obj->props[name] = v; }
napi_value mock_get(napi_value obj, const char *name) { auto it = obj->props.find(name); return it == obj->props.end() ? NULL : it->second; }
napi_value mock_call(napi_env env, napi_value fn, std::vector<napi_value> args)
{
	napi_callback_info__ info;
	info.argv = args;
	return fn->cb(env, &info);
}
// run queued threadsafe-function calls on THIS thread (the event loop); waits up to ms
int mock_run_loop(napi_env env, int ms)
{
	std::unique_lock<std::mutex> lk(env->mu);
	if (env->ready.empty())
		env->cv.wait_for(lk, std::chrono::milliseconds(ms));
	int n = 0;
	while (!env->ready.empty()) {
		napi_threadsafe_function f = env->ready.front();
		env->ready.pop_front();
		lk.unlock();
		if (f->fn && f->fn->fn) f->fn->fn();
		n++;
		lk.lock();
	}
	return n;
}
extern "C" napi_value napi_register_module_v1(napi_env env, napi_value exports);
napi_value mock_load_addon(napi_env env) { return napi_register_module_v1(env, mock_object(env)); }

// ---------------------------------------------------------------- N-API side
extern "C" {

napi_status napi_get_cb_info(napi_env, napi_callback_info info, size_t *argc, napi_value *argv,
    napi_value *this_arg, void **data)
{
	const size_t want = argc ? *argc : 0;
	for (size_t i = 0; i < want; i++) argv[i] = i < info->argv.size() ? info->argv[i] : NULL;
	if (argc) *argc = info->argv.size();
	if (this_arg) *this_arg = NULL;
	if (data) *data = NULL;
	return napi_ok;
}
napi_status napi_throw_error(napi_env env, const char *code, const char *msg)
{
	env->pending = true; env->code = code ? code : ""; env->msg = msg ? msg : "";
	return napi_ok;
}
napi_status napi_get_value_external(napi_env, napi_value v, void **result)
{
	if (!v || v->kind != MK_EXTERNAL) return napi_invalid_arg;
	*result = v->ptr; return napi_ok;
}
napi_status napi_has_named_property(napi_env, napi_value o, const char *n, bool *r)
{
	if (!o || o->kind != MK_OBJECT) return napi_object_expected;
	*r = o->props.count(n) != 0; return napi_ok;
}
napi_status napi_get_named_property(napi_env, napi_value o, const char *n, napi_value *r)
{
	if (!o || o->kind != MK_OBJECT) return napi_object_expected;
	*r = o->props[n]; return napi_ok;
}
napi_status napi_set_named_property(napi_env, napi_value o, const char *n, napi_value v)
{
	if (!o || o->kind != MK_OBJECT) return napi_object_expected;
	o->props[n] = v; return napi_ok;
}
napi_status napi_get_value_double(napi_env, napi_value v, double *r)
{
	if (!v || v->kind != MK_NUMBER) return napi_number_expected;
	*r = v->num; return napi_ok;
}
napi_status napi_get_value_uint32(napi_env, napi_value v, uint32_t *r)
{
	if (!v || v->kind != MK_NUMBER) return napi_number_expected;
	*r = (uint32_t)v->num; return napi_ok;
}
napi_status napi_create_external(napi_env env, void *data, napi_finalize, void *, napi_value *r)
{
	*r = mk(env, MK_EXTERNAL); (*r)->ptr = data; return napi_ok;
}
napi_status napi_create_external_arraybuffer(napi_env env, void *data, size_t n, napi_finalize, void *,
    napi_value *r)
{
	*r = mk(env, MK_ARRAYBUFFER); (*r)->ptr = data; (*r)->len = n; return napi_ok;
}
napi_status napi_get_buffer_info(napi_env, napi_value v, void **data, size_t *len)
{
	if (!v || v->kind != MK_BUFFER) return napi_invalid_arg;
	*data = v->ptr; *len = v->len; return napi_ok;
}
napi_status napi_get_null(napi_env env, napi_value *r) { *r = mk(env, MK_NULL); return napi_ok; }
napi_status napi_create_double(napi_env env, double d, napi_value *r) { *r = mock_number(env, d); return napi_ok; }
napi_status napi_create_int32(napi_env env, int32_t d, napi_value *r) { *r = mock_number(env, d); return napi_ok; }
napi_status napi_create_string_utf8(napi_env env, const char *s, size_t n, napi_value *r)
{
	*r = mk(env, MK_STRING);
	(*r)->str = (n == NAPI_AUTO_LENGTH) ? std::string(s) : std::string(s, n);
	return napi_ok;
}
napi_status napi_create_object(napi_env env, napi_value *r) { *r = mk(env, MK_OBJECT); return napi_ok; }
napi_status napi_create_array_with_length(napi_env env, size_t n, napi_value *r)
{
	*r = mk(env, MK_ARRAY); (*r)->elems.resize(n); return napi_ok;
}
napi_status napi_set_element(napi_env, napi_value a, uint32_t i, napi_value v)
{
	if (!a || a->kind != MK_ARRAY) return napi_array_expected;
	if (i >= a->elems.size()) a->elems.resize(i + 1);
	a->elems[i] = v; return napi_ok;
}
napi_status napi_create_bigint_uint64(napi_env env, uint64_t x, napi_value *r)
{
	*r = mk(env, MK_BIGINT); (*r)->big = x; return napi_ok;
}
napi_status napi_define_properties(napi_env env, napi_value o, size_t n, const napi_property_descriptor *d)
{
	for (size_t i = 0; i < n; i++) {
		napi_value f = mk(env, MK_FUNCTION);
		f->cb = d[i].method;
		o->props[d[i].utf8name] = f;
	}
	return napi_ok;
}
napi_status napi_create_threadsafe_function(napi_env env, napi_value func, napi_value, napi_value, size_t,
    size_t, void *, napi_finalize, void *, napi_threadsafe_function_call_js call_js,
    napi_threadsafe_function *result)
{
	if (!func || func->kind != MK_FUNCTION || call_js != NULL) return napi_invalid_arg;
	napi_threadsafe_function f = new napi_threadsafe_function__();
	f->env = env; f->fn = func;
	*result = f;
	return napi_ok;
}
napi_status napi_call_threadsafe_function(napi_threadsafe_function f, void *, napi_threadsafe_function_call_mode)
{
	std::lock_guard<std::mutex> g(f->env->mu);
	if (f->released) return napi_generic_failure;
	f->env->ready.push_back(f);
	f->env->cv.notify_all();
	return napi_ok;
}
napi_status napi_release_threadsafe_function(napi_threadsafe_function f, napi_threadsafe_function_release_mode)
{
	std::lock_guard<std::mutex> g(f->env->mu);
	f->released = true;
	return napi_ok;
}
napi_status napi_unref_threadsafe_function(napi_env, napi_threadsafe_function) { return napi_ok; }

} // extern "C"
