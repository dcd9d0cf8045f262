// napi_harness_blocks.cc -- TEST INFRASTRUCTURE: napi_harness.cc's drive of js/src/binding.cc (open,
// watch, write..., flush, peek/consume on every wake-up) with the block-check options a stage passes:
// open({... flags}) and, at the end, blockStats(h) as js/lib/gpuSnapshotStage.js publishes it.
// usage: napi_harness_blocks <mode 0..4> <flags> <input file> <output file>
// prints one JSON line with the blockStats keys; exit 0 ok, 3 = an exported function threw.
#include "napi_mock.h"
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

static napi_env env;
static napi_value addon;

static bool threw(const char *where)
{
	std::string code, msg;
	if (!mock_exception(env, &code, &msg)) return false;
	printf("{\"threw\": \"%s\", \"code\": \"%s\", \"message\": \"%s\"}\n", where, code.c_str(), msg.c_str());
	return true;
}

static napi_value call(const char *name, std::vector<napi_value> args)
{
	napi_value fn = mock_get(addon, name);
	if (fn == NULL) { fprintf(stderr, "addon has no export %s\n", name); exit(2); }
	return mock_call(env, fn, args);
}

int main(int argc, char **argv)
{
	if (argc < 5) { fprintf(stderr, "usage: %s mode flags in out\n", argv[0]); return 2; }
	FILE *fi = fopen(argv[3], "rb"), *fo = fopen(argv[4], "wb");
	if (!fi || !fo) { perror("open"); return 2; }
	fseek(fi, 0, SEEK_END);
	const size_t total = (size_t)ftell(fi);
	fseek(fi, 0, SEEK_SET);
	std::vector<uint8_t> in(total);
	if (total && fread(in.data(), 1, total, fi) != total) { perror("read"); return 2; }

	env = mock_env_new();
	addon = mock_load_addon(env);
	napi_value cfg = mock_object(env);
	mock_set(cfg, "mode", mock_number(env, atoi(argv[1])));
	mock_set(cfg, "flags", mock_number(env, atoi(argv[2])));
	mock_set(cfg, "device", mock_number(env, 0));
	mock_set(cfg, "ringBytes", mock_number(env, 8 << 20));
	mock_set(cfg, "outRingBytes", mock_number(env, 8 << 20));
	mock_set(cfg, "batchBytes", mock_number(env, 1 << 20));
	napi_value h = call("open", { cfg });
	if (threw("open")) return 3;
	napi_value watcher = call("watch", { h, mock_function(env, [] {}) });
	if (threw("watch")) return 3;

	size_t fed = 0, out_bytes = 0;
	bool flushed = false, eof = false;
	int idle = 0;
	while (!eof) {
		while (fed < total) {
			const size_t n = std::min<size_t>(1u << 20, total - fed);
			napi_value r = call("write", { h, mock_buffer(env, in.data() + fed, n) });
			if (threw("write")) { call("unwatch", { watcher }); call("close", { h }); return 3; }
			fed += (size_t)r->num;
			if ((size_t)r->num < n) break;
		}
		if (fed == total && !flushed) {
			call("flush", { h });
			if (threw("flush")) { call("unwatch", { watcher }); call("close", { h }); return 3; }
			flushed = true;
		}
		const int fired = mock_run_loop(env, 200);
		idle = fired ? 0 : idle + 1;
		if (idle > 300) { printf("{\"error\": \"no wake-up for 60 s\"}\n"); return 4; }
		for (;;) {
			napi_value ab = call("peek", { h });
			if (threw("peek")) { call("unwatch", { watcher }); call("close", { h }); return 3; }
			if (ab->kind == MK_NULL) break;
			if (ab->kind == MK_STRING && ab->str == "eof") { eof = true; break; }
			fwrite(ab->ptr, 1, ab->len, fo);
			out_bytes += ab->len;
			call("consume", { h, mock_number(env, (double)ab->len) });
			if (threw("consume")) { call("unwatch", { watcher }); call("close", { h }); return 3; }
		}
	}
	fclose(fo);
	napi_value bs = call("blockStats", { h });
	if (threw("blockStats")) return 3;
	call("unwatch", { watcher });
	call("close", { h });
	printf("{\"ok\": true, \"out\": %zu", out_bytes);
	for (const char *k : { "logicalOk", "frameOk", "frameMiss", "skipped", "lzjbEncoded", "zleEncoded", "logicalChecked",
	    "firstFrameMiss" })
		printf(", \"%s\": %.0f", k, mock_get(bs, k)->num);
	printf("}\n");
	return 0;
}
