// binding.cc -- thin N-API addon over the C ABI of libmanatee_gpu.so
// (include/manatee_gpu.h).  It adds NO logic: every export is one mtz_* call.
//
// NOT BUILT INTO A NODE ADDON HERE: the build image has no Node.js and no node_api.h
// (`node --version`: not found).  The test-suite compiles this very file against a stub of
// the N-API declarations (tests/stubs/node_api.h), links it with a miniature in-process
// N-API (tests/stubs/napi_mock.cc) and executes it through tests/stubs/napi_harness.cc --
// on the CPU with an in-memory stand-in of the library, on an H100 with the real one
// (tests/test_zz_napi_harness.py).
//
// JS surface (used by js/lib/gpuSnapshotStage.js):
//   open({mode, device, deviceMask, ringBytes, outRingBytes, batchBytes, slots}) -> handle (external)
//                                  deviceMask: bit i set = CUDA device i is part of the device group
//                                  (mtz_config.devices[]); 0 = just `device`
//   attach(handle, peer)           -> egress GPU of the peer; before the first byte (mtz_fanout_attach)
//   cancel(handle)                 -> fail the handle with MTZ_ECANCELED, wake everything (stage._destroy)
//   acquire(handle, want)          -> ArrayBuffer over the PINNED input ring slice (zero copy) | null
//   commit(handle, n)
//   write(handle, Buffer)          -> bytes accepted (non-blocking; 0 == ring full)
//   flush(handle)
//   peek(handle[, peer])           -> ArrayBuffer over the pinned output slice | null | 'eof'
//   consume(handle, n[, peer])
//   eventFd(handle)                -> the library's eventfd (readable when output / error / EOF is pending)
//   watch(handle, fn)              -> watcher (external): a small native thread poll(2)s that fd and
//                                     calls fn() ON THE EVENT LOOP through a napi_threadsafe_function,
//                                     so the loop never blocks and never busy-polls
//   unwatch(watcher)               -> stops and joins the thread (call before close)
//   stats(handle) -> {bytesIn, bytesOut, records, ...}; endChecksum(handle) -> [4 x BigInt]
//   close(handle)
// Every failing call throws Error(mtz_last_error) with .code = MTZ_E* so the stage
// can destroy(err), which the sender maps to job.done='failed' (lib/backupSender.js:218).
#include <node_api.h>
#include <poll.h>
#include <stdio.h>
#include <string.h>
#include <sys/eventfd.h>
#include <unistd.h>
#include <thread>
#include "../../include/manatee_gpu.h"

#define NAPI_OK(call) do { if ((call) != napi_ok) { napi_throw_error(env, NULL, #call); return NULL; } } while (0)

static napi_value throw_mtz(napi_env env, mtz_handle *h, int32_t rc)
{
	char code[16];
	snprintf(code, sizeof code, "%d", rc);
	const char *msg = mtz_last_error(h);
	napi_throw_error(env, code, (msg && *msg) ? msg : mtz_strerror(rc));
	return NULL;
}

static mtz_handle *get_handle(napi_env env, napi_value v)
{
	void *p = NULL;
	if (napi_get_value_external(env, v, &p) != napi_ok) return NULL;
	return (mtz_handle *)p;
}

static uint64_t get_u64_prop(napi_env env, napi_value obj, const char *name)
{
	napi_value v; bool has = false; double d = 0;
	if (napi_has_named_property(env, obj, name, &has) != napi_ok || !has) return 0;
	napi_get_named_property(env, obj, name, &v);
	napi_get_value_double(env, v, &d);
	return (uint64_t)d;
}

static napi_value Open(napi_env env, napi_callback_info info)
{
	size_t argc = 1; napi_value argv[1];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_config cfg; memset(&cfg, 0, sizeof cfg);
	cfg.struct_size = sizeof cfg;
	cfg.mode = (uint32_t)get_u64_prop(env, argv[0], "mode");
	cfg.device = (int32_t)get_u64_prop(env, argv[0], "device");
	cfg.ring_bytes = get_u64_prop(env, argv[0], "ringBytes");
	cfg.out_ring_bytes = get_u64_prop(env, argv[0], "outRingBytes");
	cfg.batch_bytes = get_u64_prop(env, argv[0], "batchBytes");
	cfg.n_slots = (uint32_t)get_u64_prop(env, argv[0], "slots");
	cfg.flags = (uint32_t)get_u64_prop(env, argv[0], "flags");
	const uint64_t mask = get_u64_prop(env, argv[0], "deviceMask");
	for (int d = 0; d < MTZ_MAX_DEVICES; d++)
		if (mask & (1ull << d)) cfg.devices[cfg.n_devices++] = d;
	mtz_handle *h = NULL;
	int32_t rc = mtz_open(&cfg, &h);
	if (rc != MTZ_OK) return throw_mtz(env, NULL, rc);
	napi_value ext;
	NAPI_OK(napi_create_external(env, h, NULL, NULL, &ext));
	return ext;
}

static void noop_finalize(napi_env, void *, void *) {}

static napi_value Acquire(napi_env env, napi_callback_info info)
{
	size_t argc = 2; napi_value argv[2];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	uint32_t want = 0; napi_get_value_uint32(env, argv[1], &want);
	void *p = NULL; size_t got = 0;
	int32_t rc = mtz_ring_acquire(h, want, &p, &got);
	napi_value out;
	if (rc == MTZ_EAGAIN) { napi_get_null(env, &out); return out; }
	if (rc != MTZ_OK) return throw_mtz(env, h, rc);
	// library-owned pinned memory: external ArrayBuffer with a no-op finalizer
	NAPI_OK(napi_create_external_arraybuffer(env, p, got, noop_finalize, NULL, &out));
	return out;
}

static napi_value Commit(napi_env env, napi_callback_info info)
{
	size_t argc = 2; napi_value argv[2];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	uint32_t n = 0; napi_get_value_uint32(env, argv[1], &n);
	int32_t rc = mtz_ring_commit(h, n);
	if (rc != MTZ_OK) return throw_mtz(env, h, rc);
	return NULL;
}

static napi_value Write(napi_env env, napi_callback_info info)
{
	size_t argc = 2; napi_value argv[2];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	void *data = NULL; size_t len = 0;
	NAPI_OK(napi_get_buffer_info(env, argv[1], &data, &len));
	// non-blocking: the event loop must never stall (SURVEY.md 8b "Threading")
	size_t done = 0;
	while (done < len) {
		void *p = NULL; size_t got = 0;
		int32_t rc = mtz_ring_acquire(h, len - done, &p, &got);
		if (rc == MTZ_EAGAIN) break;
		if (rc != MTZ_OK) return throw_mtz(env, h, rc);
		memcpy(p, (const char *)data + done, got);
		rc = mtz_ring_commit(h, got);
		if (rc != MTZ_OK) return throw_mtz(env, h, rc);
		done += got;
	}
	napi_value out; napi_create_double(env, (double)done, &out);
	return out;
}

static napi_value Flush(napi_env env, napi_callback_info info)
{
	size_t argc = 1; napi_value argv[1];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	int32_t rc = mtz_flush(h);
	if (rc != MTZ_OK) return throw_mtz(env, h, rc);
	return NULL;
}

static napi_value Attach(napi_env env, napi_callback_info info)
{
	size_t argc = 2; napi_value argv[2];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	uint32_t peer = 0; napi_get_value_uint32(env, argv[1], &peer);
	int32_t rc = mtz_fanout_attach(h, (int32_t)peer);
	if (rc < 0) return throw_mtz(env, h, rc);
	napi_value out; napi_create_int32(env, rc, &out);
	return out;
}

static napi_value Cancel(napi_env env, napi_callback_info info)
{
	size_t argc = 1; napi_value argv[1];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_cancel(get_handle(env, argv[0]));
	return NULL;
}

static napi_value Peek(napi_env env, napi_callback_info info)
{
	size_t argc = 2; napi_value argv[2];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	uint32_t peer = 0;
	if (argc >= 2) napi_get_value_uint32(env, argv[1], &peer);
	const void *p = NULL; size_t n = 0;
	int32_t rc = mtz_out_peek_peer(h, (int32_t)peer, &p, &n);
	napi_value out;
	if (rc == MTZ_EAGAIN) { napi_get_null(env, &out); return out; }
	if (rc == MTZ_EOF) { napi_create_string_utf8(env, "eof", 3, &out); return out; }
	if (rc != MTZ_OK) return throw_mtz(env, h, rc);
	NAPI_OK(napi_create_external_arraybuffer(env, (void *)p, n, noop_finalize, NULL, &out));
	return out;
}

static napi_value Consume(napi_env env, napi_callback_info info)
{
	size_t argc = 3; napi_value argv[3];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	uint32_t n = 0, peer = 0; napi_get_value_uint32(env, argv[1], &n);
	if (argc >= 3) napi_get_value_uint32(env, argv[2], &peer);
	int32_t rc = mtz_out_consume_peer(h, (int32_t)peer, n);
	if (rc != MTZ_OK) return throw_mtz(env, h, rc);
	return NULL;
}

static napi_value EventFd(napi_env env, napi_callback_info info)
{
	size_t argc = 1; napi_value argv[1];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	napi_value out; napi_create_int32(env, mtz_event_fd(h), &out);
	return out;
}

// ---- wake-up path: library eventfd -> native poll thread -> threadsafe function -> JS ----
struct Watcher {
	napi_threadsafe_function tsfn = NULL;
	std::thread th;
	int efd = -1;      // the library's eventfd (owned by the handle)
	int stop_fd = -1;  // ours: written by unwatch()
};

static void watcher_main(Watcher *w)
{
	struct pollfd fds[2];
	fds[0].fd = w->efd; fds[0].events = POLLIN;
	fds[1].fd = w->stop_fd; fds[1].events = POLLIN;
	for (;;) {
		fds[0].revents = fds[1].revents = 0;
		if (poll(fds, 2, -1) < 0) continue;                       // EINTR
		if (fds[1].revents) break;
		if (fds[0].revents & (POLLERR | POLLHUP | POLLNVAL)) break;
		if (fds[0].revents & POLLIN) {
			uint64_t v;
			if (read(w->efd, &v, sizeof v) < 0) { /* raced with another reader: fine */ }
			// default call_js: invokes the JS function with no arguments on the loop thread
			napi_call_threadsafe_function(w->tsfn, NULL, napi_tsfn_nonblocking);
		}
	}
	napi_release_threadsafe_function(w->tsfn, napi_tsfn_release);
}

static void watcher_stop(Watcher *w)
{
	if (w->stop_fd >= 0) {
		const uint64_t one = 1;
		if (write(w->stop_fd, &one, sizeof one) < 0) { /* thread exits on POLLNVAL at close */ }
		if (w->th.joinable()) w->th.join();
		close(w->stop_fd);
		w->stop_fd = -1;
	}
}

// the Watcher lives as long as its JS external: unwatch() stops the thread, GC frees the struct
static void watcher_finalize(napi_env, void *data, void *)
{
	Watcher *w = (Watcher *)data;
	watcher_stop(w);
	delete w;
}

static napi_value Watch(napi_env env, napi_callback_info info)
{
	size_t argc = 2; napi_value argv[2];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	const int32_t efd = mtz_event_fd(h);
	if (efd < 0) return throw_mtz(env, h, efd);
	Watcher *w = new Watcher();
	w->efd = efd;
	w->stop_fd = eventfd(0, EFD_CLOEXEC);
	napi_value name;
	NAPI_OK(napi_create_string_utf8(env, "manatee-gpu-wakeup", NAPI_AUTO_LENGTH, &name));
	if (w->stop_fd < 0 ||
	    napi_create_threadsafe_function(env, argv[1], NULL, name, 0, 1, NULL, NULL, NULL, NULL,
	    &w->tsfn) != napi_ok) {
		if (w->stop_fd >= 0) close(w->stop_fd);
		delete w;
		napi_throw_error(env, NULL, "cannot create the wake-up function");
		return NULL;
	}
	// the stage keeps the loop alive through its stream state, not through this function
	napi_unref_threadsafe_function(env, w->tsfn);
	w->th = std::thread(watcher_main, w);
	napi_value ext;
	NAPI_OK(napi_create_external(env, w, watcher_finalize, NULL, &ext));
	return ext;
}

static napi_value Unwatch(napi_env env, napi_callback_info info)
{
	size_t argc = 1; napi_value argv[1];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	void *p = NULL;
	if (napi_get_value_external(env, argv[0], &p) != napi_ok || p == NULL) return NULL;
	watcher_stop((Watcher *)p);
	return NULL;
}

static napi_value Stats(napi_env env, napi_callback_info info)
{
	size_t argc = 1; napi_value argv[1];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	mtz_stats st;
	int32_t rc = mtz_get_stats(h, &st);
	if (rc != MTZ_OK) return throw_mtz(env, h, rc);
	napi_value o, v; napi_create_object(env, &o);
#define PUT(name, field) napi_create_double(env, (double)st.field, &v); napi_set_named_property(env, o, name, v)
	PUT("bytesIn", bytes_in); PUT("bytesOut", bytes_out); PUT("records", records);
	PUT("writeRecords", write_records); PUT("lz4Decoded", lz4_decoded); PUT("lz4Encoded", lz4_encoded);
	PUT("batches", batches); PUT("gpuMs", gpu_ms); PUT("kernelLaunches", kernel_launches);
	PUT("lz4Certified", lz4_certified);
#undef PUT
	return o;
}

// block-checksum counters (MTZ_FLAG_BLOCK_CKSUM): job.gpu.blocks.  A weak reference: the addon
// still loads against a libmanatee_gpu.so older than the entry point (the ABI only grows), and
// blockStats() returns undefined there.
#pragma weak mtz_get_block_stats
static napi_value BlockStats(napi_env env, napi_callback_info info)
{
	size_t argc = 1; napi_value argv[1];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	if (mtz_get_block_stats == NULL) return NULL;
	mtz_block_stats st; memset(&st, 0, sizeof st);
	st.struct_size = sizeof st;
	int32_t rc = mtz_get_block_stats(h, &st);
	if (rc != MTZ_OK) return throw_mtz(env, h, rc);
	napi_value o, v; napi_create_object(env, &o);
#define PUT(name, field) napi_create_double(env, (double)st.field, &v); napi_set_named_property(env, o, name, v)
	PUT("logicalOk", logical_ok); PUT("frameOk", frame_ok); PUT("frameMiss", frame_miss);
	PUT("skipped", skipped);
	PUT("sha256", sha256);      // an older library fills fewer bytes: 0 from the memset
	PUT("sha512", sha512);
	PUT("framesEncoded", frames_encoded);
	PUT("lzjbEncoded", lzjb_encoded);
	PUT("zleEncoded", zle_encoded);
#undef PUT
	// ~0 (no miss) does not survive a double: -1 says "none"
	napi_create_double(env, st.first_frame_miss == ~0ull ? -1.0 : (double)st.first_frame_miss, &v);
	napi_set_named_property(env, o, "firstFrameMiss", v);
	return o;
}

static napi_value EndChecksum(napi_env env, napi_callback_info info)
{
	size_t argc = 1; napi_value argv[1];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_handle *h = get_handle(env, argv[0]);
	uint64_t ck[4] = { 0, 0, 0, 0 };
	int32_t rc = mtz_end_checksum(h, ck);
	if (rc != MTZ_OK) return throw_mtz(env, h, rc);
	napi_value arr, v;
	NAPI_OK(napi_create_array_with_length(env, 4, &arr));
	for (uint32_t i = 0; i < 4; i++) {
		NAPI_OK(napi_create_bigint_uint64(env, ck[i], &v));   // 64-bit words do not fit a double
		NAPI_OK(napi_set_element(env, arr, i, v));
	}
	return arr;
}

static napi_value Close(napi_env env, napi_callback_info info)
{
	size_t argc = 1; napi_value argv[1];
	NAPI_OK(napi_get_cb_info(env, info, &argc, argv, NULL, NULL));
	mtz_close(get_handle(env, argv[0]));
	return NULL;
}

static napi_value Init(napi_env env, napi_value exports)
{
	napi_property_descriptor d[] = {
		{"open", 0, Open, 0, 0, 0, napi_default, 0}, {"acquire", 0, Acquire, 0, 0, 0, napi_default, 0},
		{"commit", 0, Commit, 0, 0, 0, napi_default, 0}, {"write", 0, Write, 0, 0, 0, napi_default, 0},
		{"flush", 0, Flush, 0, 0, 0, napi_default, 0}, {"peek", 0, Peek, 0, 0, 0, napi_default, 0},
		{"consume", 0, Consume, 0, 0, 0, napi_default, 0}, {"eventFd", 0, EventFd, 0, 0, 0, napi_default, 0},
		{"stats", 0, Stats, 0, 0, 0, napi_default, 0}, {"close", 0, Close, 0, 0, 0, napi_default, 0},
		{"blockStats", 0, BlockStats, 0, 0, 0, napi_default, 0},
		{"endChecksum", 0, EndChecksum, 0, 0, 0, napi_default, 0},
		{"watch", 0, Watch, 0, 0, 0, napi_default, 0}, {"unwatch", 0, Unwatch, 0, 0, 0, napi_default, 0},
		{"attach", 0, Attach, 0, 0, 0, napi_default, 0}, {"cancel", 0, Cancel, 0, 0, 0, napi_default, 0},
	};
	napi_define_properties(env, exports, sizeof d / sizeof d[0], d);
	return exports;
}

NAPI_MODULE(manatee_gpu, Init)
