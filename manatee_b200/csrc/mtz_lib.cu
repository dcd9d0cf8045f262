// mtz_lib.cu -- C-ABI entry points of libmanatee_gpu.so (include/manatee_gpu.h).
//
// Replaces the data path of the reference's two pipes,
//   zfsSend.stdout.pipe(socket)      lib/backupSender.js:179
//   socket.pipe(zfsRecv.stdin)       lib/zfsClient.js:826
// with: pinned host ring -> cudaMemcpyAsync -> HBM -> sm_90a kernels
// (Fletcher-4 verify / LZ4 decode / LZ4 encode / re-stamp) -> pinned ring.
// There is NO CPU fallback: without a usable device mtz_open fails MTZ_ENOGPU.
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <algorithm>
#include "mtz_internal.h"

using namespace mtz;

static thread_local std::string g_open_err;

namespace mtz {

int32_t fail(mtz_handle *h, int32_t code, const char *fmt, ...)
{
	char buf[512];
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(buf, sizeof buf, fmt, ap);
	va_end(ap);
	if (h) {
		{
			// message and code are set together, once, under the lock: a second failure on
			// another thread never overwrites the string mtz_last_error() handed out
			std::lock_guard<std::mutex> g(h->err_mu);
			if (h->failed.load() == 0) {
				h->err = buf;
				h->failed.store(code);
			}
		}
		engine_wake_all(h);
	} else {
		g_open_err = buf;
	}
	return code;
}

int32_t fail_cuda(mtz_handle *h, cudaError_t e, const char *what)
{
	return fail(h, MTZ_ECUDA, "CUDA error %d (%s) at %s", (int)e,
	    cudaGetErrorString(e), what);
}

} // namespace mtz

#define CHECK_H(h)                                                             \
	do {                                                                       \
		if ((h) == nullptr) return MTZ_EINVAL;                                 \
		int32_t f__ = (h)->failed.load();                                      \
		if (f__ != 0) return f__;                                              \
	} while (0)

extern "C" {

int32_t mtz_abi_version(void) { return MTZ_ABI_VERSION; }

const char *mtz_strerror(int32_t code)
{
	switch (code) {
	case MTZ_OK: return "ok";
	case MTZ_EINVAL: return "invalid argument or state";
	case MTZ_EAGAIN: return "would block";
	case MTZ_ECUDA: return "CUDA failure";
	case MTZ_EFORMAT: return "malformed ZFS send stream";
	case MTZ_ECKSUM: return "stream checksum mismatch";
	case MTZ_ECODEC: return "LZ4 frame does not decode";
	case MTZ_ENOSPC: return "output capacity exceeded";
	case MTZ_ENOMEM: return "out of memory";
	case MTZ_EOF: return "end of stream";
	case MTZ_ENOGPU: return "no sm_90 GPU (no CPU fallback exists)";
	default: return "unknown error";
	}
}

const char *mtz_last_error(mtz_handle *h)
{
	if (h == nullptr) return g_open_err.c_str();
	// h->err is written exactly once (fail()), so the pointer stays valid until mtz_close
	std::lock_guard<std::mutex> g(h->err_mu);
	return h->err.c_str();
}

int32_t mtz_device_count(void)
{
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess) { (void)cudaGetLastError(); return 0; }
	int ok = 0;
	for (int i = 0; i < n; i++) {
		cudaDeviceProp p;
		if (cudaGetDeviceProperties(&p, i) == cudaSuccess && p.major == 9 && p.minor == 0) ok++;
	}
	return ok;
}

// ------------------------------------------------------------------ parse --
static inline uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static inline uint64_t rd64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }

// Payload sizing per record type (DRR header classify, K4's host half):
// restated from sys/zfs_ioctl.h DRR_*_PAYLOAD_SIZE ([EXTERNAL], SURVEY App. A.1).
static int64_t drr_payload(const uint8_t *h, uint32_t *lsize, uint32_t *comp)
{
	// Every record of a send stream starts 8-byte aligned (dump_bytes()/receive_read() keep
	// lengths at multiples of 8); the kernels rely on it for their 64-bit header loads, so a
	// payload length that would break it is a format error here, never a misaligned access.
	const uint32_t type = rd32(h);
	*lsize = 0; *comp = 0;
	switch (type) {
	case 0: /* BEGIN */
		if (rd64(h + 8) != 0x2F5bacbacULL) return -1;
		if (rd32(h + 4) & 7u) return -1;
		return (int64_t)rd32(h + 4);
	case 1: /* OBJECT */
		return (int64_t)(((uint64_t)rd32(h + 28) + 7) & ~7ull);
	case 3: { /* WRITE */
		const uint64_t ls = rd64(h + 32);
		const uint64_t l = h[50] ? rd64(h + 96) : ls;
		// the logical size becomes a payload length in DECOMPRESS / RECOMPRESS output, so it
		// has to keep records 8-byte aligned too (ZFS block sizes are multiples of 512)
		if (l > (1ull << 30) || (l & 7) || ls > (1ull << 30) || (ls & 7)) return -1;
		*lsize = (uint32_t)ls; *comp = h[50];
		return (int64_t)l;
	}
	case 7: { /* SPILL */
		const uint64_t l = rd64(h + 16);
		if (l > (1ull << 30) || (l & 7)) return -1;
		return (int64_t)l;
	}
	case 8: /* WRITE_EMBEDDED */
		return (int64_t)(((uint64_t)rd32(h + 52) + 7) & ~7ull);
	case 2: case 4: case 5: case 6:
		return 0;
	default:
		return -1;
	}
}

int32_t mtz_index_host(const void *buf, size_t n, mtz_rec *recs, size_t cap,
    size_t *nrec, size_t *consumed)
{
	const uint8_t *s = (const uint8_t *)buf;
	size_t off = 0, cnt = 0;
	int32_t rc = MTZ_OK;
	if (buf == nullptr && n != 0) return MTZ_EINVAL;
	while (n - off >= DRR_HDR) {
		uint32_t ls, comp;
		const int64_t pl = drr_payload(s + off, &ls, &comp);
		if (pl < 0) { rc = MTZ_EFORMAT; break; }
		if ((uint64_t)pl > n - off - DRR_HDR) break;     // incomplete record
		if (recs != nullptr) {
			if (cnt >= cap) { rc = MTZ_ENOSPC; break; }
			mtz_rec r;
			r.off = off; r.payload = (uint32_t)pl; r.type = rd32(s + off);
			r.lsize = ls; r.comp = comp; r.resv = 0;
			recs[cnt] = r;
		}
		cnt++;
		off += DRR_HDR + (size_t)pl;
	}
	if (nrec) *nrec = cnt;
	if (consumed) *consumed = off;
	return rc;
}

// ------------------------------------------------------------- lifecycle --
// Stream priorities (experiment, off by default: MTZ_STREAM_PRIORITIES=1).  The LZ4 encoder owns the
// machine for tens of milliseconds per launch; with priorities on, its streams get the LEAST
// priority and every other library stream the GREATEST, so that short kernels (plan, decode of the
// next sub-batch, assemble, the stamp chain, the NCCL broadcast) are placed the moment an encoder
// CTA retires.  The encoder is throughput-bound, so whatever runs beside it takes its issue slots
// either way; launching K2/K3 as many short-lived CTAs rather than one persistent wave (lz4_grid)
// is the default.
static bool stream_priorities()
{
	static const bool on = [] { const char *e = getenv("MTZ_STREAM_PRIORITIES"); return e != nullptr && atoi(e) != 0; }();
	return on;
}
static cudaError_t make_stream(cudaStream_t *st, bool high)
{
	int least = 0, greatest = 0;
	if (stream_priorities()) {
		cudaError_t e = cudaDeviceGetStreamPriorityRange(&least, &greatest);
		if (e != cudaSuccess) return e;
	}
	return cudaStreamCreateWithPriority(st, cudaStreamNonBlocking, high ? greatest : least);
}

static int32_t alloc_slot(mtz_handle *h, Slot &s, int di, size_t cap, size_t rec_cap)
{
	s.cap = cap; s.rec_cap = rec_cap; s.di = di;
	MTZ_CU(h, cudaSetDevice(h->devs[di].device));
	MTZ_CU(h, cudaMalloc(&s.d_in, cap + 512));
	MTZ_CU(h, cudaMalloc(&s.d_recs, rec_cap * sizeof(mtz_rec)));
	MTZ_CU(h, cudaHostAlloc(&s.h_recs, rec_cap * sizeof(mtz_rec), cudaHostAllocPortable));
	MTZ_CU(h, cudaMalloc(&s.d_sums, rec_cap * sizeof(RecSums)));
	MTZ_CU(h, cudaMalloc(&s.d_tiles, (rec_cap / SCAN_TILE + 2) * sizeof(Part)));
	MTZ_CU(h, cudaMalloc(&s.d_res, sizeof(ScanResult)));
	MTZ_CU(h, cudaHostAlloc(&s.h_res, sizeof(ScanResult), cudaHostAllocPortable));
	if (h->cfg.flags & MTZ_FLAG_BLOCK_CKSUM) {
		MTZ_CU(h, cudaMalloc(&s.d_bres, sizeof(BlockResult)));
		MTZ_CU(h, cudaHostAlloc(&s.h_bres, sizeof(BlockResult), cudaHostAllocPortable));
	}
	MTZ_CU(h, make_stream(&s.st, true));
	if (stream_priorities() && (h->cfg.mode == MTZ_MODE_COMPRESS || h->cfg.mode == MTZ_MODE_RECOMPRESS))
		MTZ_CU(h, make_stream(&s.st_k3, false));
	MTZ_CU(h, cudaEventCreateWithFlags(&s.ev_scan, cudaEventDisableTiming));
	MTZ_CU(h, cudaEventCreateWithFlags(&s.ev_h2d, cudaEventDisableTiming));
	MTZ_CU(h, cudaEventCreate(&s.ev_k3a));
	MTZ_CU(h, cudaEventCreate(&s.ev_k3b));
	MTZ_CU(h, cudaEventCreate(&s.ev_start));
	MTZ_CU(h, cudaEventCreate(&s.ev_done));
	MTZ_CU(h, cudaEventCreate(&s.ev_k1a));
	MTZ_CU(h, cudaEventCreate(&s.ev_k1b));
	MTZ_CU(h, cudaEventCreate(&s.ev_c0));
	MTZ_CU(h, cudaEventCreate(&s.ev_c1));
	return MTZ_OK;
}

static void codec_free(CodecBufs &cb);

static void free_slot(Slot &s)
{
	if (s.d_in) cudaFree(s.d_in);
	if (s.d_out) cudaFree(s.d_out);
	if (s.d_recs) cudaFree(s.d_recs);
	if (s.h_recs) cudaFreeHost(s.h_recs);
	if (s.d_sums) cudaFree(s.d_sums);
	if (s.d_tiles) cudaFree(s.d_tiles);
	if (s.d_res) cudaFree(s.d_res);
	if (s.h_res) cudaFreeHost(s.h_res);
	if (s.d_bres) cudaFree(s.d_bres);
	if (s.h_bres) cudaFreeHost(s.h_bres);
	if (s.st) cudaStreamDestroy(s.st);
	if (s.st_k3) cudaStreamDestroy(s.st_k3);
	if (s.ev_start) cudaEventDestroy(s.ev_start);
	if (s.ev_done) cudaEventDestroy(s.ev_done);
	if (s.ev_k1a) cudaEventDestroy(s.ev_k1a);
	if (s.ev_k1b) cudaEventDestroy(s.ev_k1b);
	if (s.ev_c0) cudaEventDestroy(s.ev_c0);
	if (s.ev_c1) cudaEventDestroy(s.ev_c1);
	if (s.ev_scan) cudaEventDestroy(s.ev_scan);
	if (s.ev_h2d) cudaEventDestroy(s.ev_h2d);
	if (s.ev_k3a) cudaEventDestroy(s.ev_k3a);
	if (s.ev_k3b) cudaEventDestroy(s.ev_k3b);
	codec_free(s.cb);
	s = Slot();
}

#define MAX_RECORD_BYTES ((size_t)(16u << 20) + 4096)

static int32_t k3_set_attributes(mtz_handle *h);
static int32_t launch_k2(mtz_handle *h, cudaStream_t st, const void *d_src, void *d_dst, mtz_job *d_jobs,
    uint32_t njobs, const mtz_job *seq_jobs = nullptr, uint32_t *seq_n = nullptr);

int32_t mtz_open(const mtz_config *cfg, mtz_handle **out)
{
	if (cfg == nullptr || out == nullptr) return fail(nullptr, MTZ_EINVAL, "null argument");
	*out = nullptr;
	if (cfg->struct_size < sizeof(uint32_t) * 4)
		return fail(nullptr, MTZ_EINVAL, "mtz_config.struct_size too small");
	if (cfg->mode > MTZ_MODE_PASSTHROUGH)
		return fail(nullptr, MTZ_EINVAL, "unknown mode %u", cfg->mode);
	int ndev = 0;
	cudaError_t e = cudaGetDeviceCount(&ndev);
	if (e != cudaSuccess || ndev == 0) {
		(void)cudaGetLastError();
		return fail(nullptr, MTZ_ENOGPU, "no CUDA device: %s (there is no CPU fallback)",
		    cudaGetErrorString(e));
	}
	// the device group: v1 callers (struct_size ends before n_devices) and n_devices == 0 get
	// the single `device`
	mtz_config full;
	memset(&full, 0, sizeof full);
	memcpy(&full, cfg, std::min((size_t)cfg->struct_size, sizeof full));
	if (full.n_devices > MTZ_MAX_DEVICES)
		return fail(nullptr, MTZ_EINVAL, "n_devices %u exceeds %d", full.n_devices, MTZ_MAX_DEVICES);
	if (full.n_devices == 0) { full.n_devices = 1; full.devices[0] = full.device; }
	full.device = full.devices[0];
	std::vector<cudaDeviceProp> props(full.n_devices);
	for (uint32_t i = 0; i < full.n_devices; i++) {
		const int d = full.devices[i];
		if (d < 0 || d >= ndev)
			return fail(nullptr, MTZ_EINVAL, "device %d out of range (%d visible)", d, ndev);
		for (uint32_t k = 0; k < i; k++)
			if (full.devices[k] == d) return fail(nullptr, MTZ_EINVAL, "device %d listed twice", d);
		if (cudaGetDeviceProperties(&props[i], d) != cudaSuccess || props[i].major != 9 || props[i].minor != 0)
			return fail(nullptr, MTZ_ENOGPU, "device %d is sm_%d%d; this library is built for sm_90a only",
			    d, props[i].major, props[i].minor);
	}
	if (full.n_devices > 1 && (full.flags & MTZ_FLAG_DEFER_VERIFY))
		return fail(nullptr, MTZ_EINVAL, "a device group verifies in stream order; DEFER_VERIFY is the "
		    "one-GPU-per-process shard form");
	if ((full.flags & MTZ_FLAG_BLOCK_CKSUM) && full.mode == MTZ_MODE_PASSTHROUGH)
		return fail(nullptr, MTZ_EINVAL, "PASSTHROUGH parses no record: BLOCK_CKSUM needs another mode");
	if ((full.flags & MTZ_FLAG_BLOCK_SHA256) && !(full.flags & MTZ_FLAG_BLOCK_CKSUM))
		return fail(nullptr, MTZ_EINVAL, "BLOCK_SHA256 extends the block check: it needs BLOCK_CKSUM");
	if ((full.flags & MTZ_FLAG_BLOCK_SHA512) && !(full.flags & MTZ_FLAG_BLOCK_CKSUM))
		return fail(nullptr, MTZ_EINVAL, "BLOCK_SHA512 extends the block check: it needs BLOCK_CKSUM");
	if ((full.flags & MTZ_FLAG_BLOCK_FRAMES) && !(full.flags & MTZ_FLAG_BLOCK_CKSUM))
		return fail(nullptr, MTZ_EINVAL, "BLOCK_FRAMES extends the block check: it needs BLOCK_CKSUM");
	if ((full.flags & MTZ_FLAG_BLOCK_LZJB) && !(full.flags & MTZ_FLAG_BLOCK_CKSUM))
		return fail(nullptr, MTZ_EINVAL, "BLOCK_LZJB extends the block check: it needs BLOCK_CKSUM");
	if ((full.flags & MTZ_FLAG_BLOCK_LOGICAL) && !(full.flags & MTZ_FLAG_BLOCK_CKSUM))
		return fail(nullptr, MTZ_EINVAL, "BLOCK_LOGICAL extends the block check: it needs BLOCK_CKSUM");
	if ((full.flags & MTZ_FLAG_GZIP_IN) && !(full.flags & MTZ_FLAG_COMPRESSED_IN))
		return fail(nullptr, MTZ_EINVAL, "GZIP_IN extends COMPRESSED_IN: it needs COMPRESSED_IN");
	if ((full.flags & MTZ_FLAG_GZIP_WIRE) && (full.flags & MTZ_FLAG_GZIP_IN))
		return fail(nullptr, MTZ_EINVAL, "GZIP_WIRE forwards the gzip records GZIP_IN inflates: set one of them");
	if ((full.flags & MTZ_FLAG_GZIP_WIRE) && full.mode == MTZ_MODE_COMPRESS && !(full.flags & MTZ_FLAG_COMPRESSED_IN))
		return fail(nullptr, MTZ_EINVAL, "COMPRESS: GZIP_WIRE extends COMPRESSED_IN: it needs COMPRESSED_IN");
	if ((full.flags & MTZ_FLAG_GZIP_ENCODE) && (full.flags & MTZ_FLAG_LZ4_HC))
		return fail(nullptr, MTZ_EINVAL, "GZIP_ENCODE re-codes K3's parse and LZ4_HC replaces K3: set one of them");
	if ((full.flags & MTZ_FLAG_GZIP_ENCODE) && (full.flags & MTZ_FLAG_GZIP_IN))
		return fail(nullptr, MTZ_EINVAL, "GZIP_ENCODE with gzip input: forward the gzip records with GZIP_WIRE "
		    "instead of GZIP_IN");
	const cudaDeviceProp &prop = props[0];

	mtz_handle *h = new (std::nothrow) mtz_handle();
	if (h == nullptr) return fail(nullptr, MTZ_ENOMEM, "handle allocation");
	h->cfg = full;
	const bool codec_mode = cfg->mode == MTZ_MODE_COMPRESS || cfg->mode == MTZ_MODE_DECOMPRESS ||
	    cfg->mode == MTZ_MODE_RECOMPRESS;
	// the LZ4 kernels want thousands of records in flight (one warp per record, ~5 ms per
	// record): measured e2e RECOMPRESS 26 / 41 / 48 / 49 GiB/s logical at 64 / 128 / 256 /
	// 512 MiB batches; Fletcher alone is happy with 32 MiB batches.  VERIFY with MTZ_FLAG_BLOCK_FRAMES
	// runs the same encoder over the batch's raw LZ4-keyed records, and wants its records in flight too;
	// so do the lzjb / zle encoders of MTZ_FLAG_BLOCK_LZJB (one warp per record as well)
	const bool frames_verify = cfg->mode == MTZ_MODE_VERIFY &&
	    (full.flags & (MTZ_FLAG_BLOCK_FRAMES | MTZ_FLAG_BLOCK_LZJB));
	if (h->cfg.batch_bytes == 0)
		h->cfg.batch_bytes = (codec_mode || frames_verify) ? (256ull << 20) : (32ull << 20);
	// the input ring holds the batch being filled plus the ones whose H2D copy is still pending
	if (h->cfg.ring_bytes == 0) h->cfg.ring_bytes = std::max<uint64_t>(256ull << 20, (codec_mode ? 3 : 2) * h->cfg.batch_bytes);
	if (h->cfg.out_ring_bytes == 0) h->cfg.out_ring_bytes = h->cfg.ring_bytes;
	if (h->cfg.record_bytes == 0) h->cfg.record_bytes = 131072;
	if (h->cfg.n_slots == 0) h->cfg.n_slots = 4;
	if (h->cfg.n_slots > 16) h->cfg.n_slots = 16;
	h->device = full.device;
	h->sm_count = prop.multiProcessorCount;
	h->stats.bad_record = ~0ull;
	h->devs.resize(full.n_devices);

	int32_t rc = MTZ_OK;
	auto init = [&]() -> int32_t {
		// every GPU of the group: its copy of the running checksums, the K3 attributes (they
		// are per device) and peer access for the 64-byte checksum hop
		for (size_t i = h->devs.size(); i-- > 0;) {
			DevCtx &dc = h->devs[i];
			dc.device = full.devices[i];
			dc.sm_count = props[i].multiProcessorCount;
			MTZ_CU(h, cudaSetDevice(dc.device));
			MTZ_CU(h, cudaMalloc(&dc.d_carry_in, sizeof(Ck4)));
			MTZ_CU(h, cudaMalloc(&dc.d_carry_out, sizeof(Ck4)));
			MTZ_CU(h, cudaMemset(dc.d_carry_in, 0, sizeof(Ck4)));
			MTZ_CU(h, cudaMemset(dc.d_carry_out, 0, sizeof(Ck4)));
			int32_t r = k3_set_attributes(h);
			if (r != MTZ_OK) return r;
			for (size_t k = 0; k < h->devs.size(); k++) {
				if (k == i) continue;
				int can = 0;
				if (cudaDeviceCanAccessPeer(&can, dc.device, full.devices[k]) == cudaSuccess && can) {
					cudaError_t pe = cudaDeviceEnablePeerAccess(full.devices[k], 0);
					if (pe != cudaSuccess) (void)cudaGetLastError();     // already enabled: fine
				}
			}
		}
		// the loop ends on devs[0]: the device-resident API lives there
		h->d_carry_in = h->devs[0].d_carry_in;
		h->d_carry_out = h->devs[0].d_carry_out;
		MTZ_CU(h, cudaStreamCreateWithFlags(&h->st, cudaStreamNonBlocking));
		MTZ_CU(h, cudaHostAlloc(&h->h_carry, 4 * sizeof(Ck4), cudaHostAllocPortable));
		MTZ_CU(h, cudaMalloc(&h->dv_res, sizeof(ScanResult)));
		MTZ_CU(h, cudaHostAlloc(&h->dv_hres, sizeof(ScanResult), cudaHostAllocPortable));
		MTZ_CU(h, cudaEventCreate(&h->dv_k1a));
		MTZ_CU(h, cudaEventCreate(&h->dv_k1b));
		if (full.flags & MTZ_FLAG_BLOCK_CKSUM) {
			MTZ_CU(h, cudaMalloc(&h->dv_bres, sizeof(BlockResult)));
			MTZ_CU(h, cudaHostAlloc(&h->dv_hbres, sizeof(BlockResult), cudaHostAllocPortable));
			h->bstats.first_frame_miss = ~0ull;
		}
		return MTZ_OK;
	};
	rc = init();
	if (rc != MTZ_OK) {
		g_open_err = h->err;
		mtz_close(h);
		return rc;
	}
	*out = h;
	return MTZ_OK;
}

static void engine_destroy(mtz_handle *h);
static void fanout_destroy(mtz_handle *h);

int32_t mtz_close(mtz_handle *h)
{
	if (h == nullptr) return MTZ_EINVAL;
	cudaSetDevice(h->device);
	engine_destroy(h);
	for (auto &dc : h->devs) { cudaSetDevice(dc.device); cudaDeviceSynchronize(); }
	fanout_destroy(h);
	if (h->xcomm && h->xcomm_owned) ncclCommDestroy(h->xcomm);
	cudaSetDevice(h->device);
	if (h->d_xagg) cudaFree(h->d_xagg);
	if (h->d_xall) cudaFree(h->d_xall);
	if (h->d_xbase) cudaFree(h->d_xbase);
	for (cudaEvent_t e : h->dv_k3ev) cudaEventDestroy(e);
	if (h->dv_c0) cudaEventDestroy(h->dv_c0);
	if (h->dv_c1) cudaEventDestroy(h->dv_c1);
	if (h->dv_cb2.cr != nullptr) {
		// results / offset are shared with dv_cb: do not free them twice
		h->dv_cb2.d_cres = nullptr; h->dv_cb2.d_ores = nullptr; h->dv_cb2.d_outpos = nullptr;
		h->dv_cb2.h_cres = nullptr; h->dv_cb2.h_ores = nullptr;
		codec_free(h->dv_cb2);
	}
	codec_free(h->dv_cb);
	if (h->k_hc_tab) cudaFree(h->k_hc_tab);
	if (h->k_gz_lz) cudaFree(h->k_gz_lz);
	if (h->st_post) cudaStreamDestroy(h->st_post);
	if (h->st_dec) cudaStreamDestroy(h->st_dec);
	for (int i = 0; i < 2; i++) {
		if (h->ev_dec[i]) cudaEventDestroy(h->ev_dec[i]);
		if (h->ev_pre[i]) cudaEventDestroy(h->ev_pre[i]);
		if (i == 0 && h->ev_reset) cudaEventDestroy(h->ev_reset);
		if (h->ev_post[i]) cudaEventDestroy(h->ev_post[i]);
	}
	if (h->dv_all_orecs) cudaFree(h->dv_all_orecs);
	if (h->dv_all_osums) cudaFree(h->dv_all_osums);
	if (h->dv_all_steps) cudaFree(h->dv_all_steps);
	if (h->d_ires) cudaFree(h->d_ires);
	if (h->d_ishared) cudaFree(h->d_ishared);
	if (h->h_ires) cudaFreeHost(h->h_ires);
	if (h->dv_k1a) cudaEventDestroy(h->dv_k1a);
	if (h->dv_k1b) cudaEventDestroy(h->dv_k1b);
	if (h->dv_bres) cudaFree(h->dv_bres);
	if (h->dv_hbres) cudaFreeHost(h->dv_hbres);
	for (auto &s : h->slots) { cudaSetDevice(h->devs[s.di].device); free_slot(s); }
	cudaSetDevice(h->device);
	if (h->dv_sums) cudaFree(h->dv_sums);
	if (h->dv_tiles) cudaFree(h->dv_tiles);
	if (h->dv_res) cudaFree(h->dv_res);
	if (h->dv_hres) cudaFreeHost(h->dv_hres);
	if (h->h_carry) cudaFreeHost(h->h_carry);
	if (h->st) cudaStreamDestroy(h->st);
	for (auto &dc : h->devs) {
		cudaSetDevice(dc.device);
		if (dc.d_carry_in) cudaFree(dc.d_carry_in);
		if (dc.d_carry_out) cudaFree(dc.d_carry_out);
	}
	delete h;
	return MTZ_OK;
}

int32_t mtz_get_stats(mtz_handle *h, mtz_stats *st)
{
	if (h == nullptr || st == nullptr) return MTZ_EINVAL;
	std::lock_guard<std::mutex> g(h->stats_mu);
	*st = h->stats;
	return MTZ_OK;
}

int32_t mtz_get_block_stats(mtz_handle *h, mtz_block_stats *st)
{
	if (h == nullptr || st == nullptr || st->struct_size < 2 * sizeof(uint32_t)) return MTZ_EINVAL;
	mtz_block_stats b;
	memset(&b, 0, sizeof b);
	if (h->cfg.flags & MTZ_FLAG_BLOCK_CKSUM) {
		std::lock_guard<std::mutex> g(h->stats_mu);
		b = h->bstats;
	}
	const size_t n = std::min((size_t)st->struct_size, sizeof b);
	b.struct_size = (uint32_t)n;
	memcpy(st, &b, n);
	return MTZ_OK;
}

int32_t mtz_get_compressed_in_stats(mtz_handle *h, mtz_compressed_in_stats *st)
{
	if (h == nullptr || st == nullptr || st->struct_size < 2 * sizeof(uint32_t)) return MTZ_EINVAL;
	mtz_compressed_in_stats c;
	{
		std::lock_guard<std::mutex> g(h->stats_mu);
		c = h->cstats;
	}
	const size_t n = std::min((size_t)st->struct_size, sizeof c);
	c.struct_size = (uint32_t)n; c.pad = 0;
	memcpy(st, &c, n);
	return MTZ_OK;
}

int32_t mtz_end_checksum(mtz_handle *h, uint64_t out[4])
{
	if (h == nullptr || out == nullptr) return MTZ_EINVAL;
	std::lock_guard<std::mutex> g(h->stats_mu);
	if (!h->stats.end_seen) return MTZ_EAGAIN;
	memcpy(out, h->end_ck, 32);
	return MTZ_OK;
}

int32_t mtz_host_alloc(size_t bytes, void **ptr)
{
	if (ptr == nullptr) return MTZ_EINVAL;
	cudaError_t e = cudaHostAlloc(ptr, bytes, cudaHostAllocPortable);
	if (e != cudaSuccess) { (void)cudaGetLastError(); *ptr = nullptr; return MTZ_ENOMEM; }
	return MTZ_OK;
}

int32_t mtz_host_free(void *ptr)
{
	if (ptr == nullptr) return MTZ_OK;
	return cudaFreeHost(ptr) == cudaSuccess ? MTZ_OK : MTZ_ECUDA;
}

// ------------------------------------------------------- kernel launches --
static inline void count_launch(mtz_handle *h, uint64_t n)
{
	std::lock_guard<std::mutex> g(h->stats_mu);
	h->stats.kernel_launches += n;
}

// lanes per record by average record size: small records share a warp
static void launch_k1_kernel(mtz_handle *h, cudaStream_t st, const uint8_t *d_in, const mtz_rec *d_recs,
    size_t nrec, RecSums *d_sums, uint32_t body_from, size_t avg_rec)
{
	const size_t cap = (size_t)h->sm_count * K1_MINBLOCKS * 8;
	if (avg_rec >= (96u << 10)) {
		const unsigned grid = (unsigned)std::min<size_t>((nrec + K1_WARPS - 1) / K1_WARPS, cap);
		k1_record_sums<<<grid, K1_THREADS, 0, st>>>(d_in, d_recs, (uint32_t)nrec, d_sums, body_from);
	} else if (avg_rec >= (24u << 10)) {
		const unsigned grid = (unsigned)std::min<size_t>((nrec + K1_WARPS * 2 - 1) / (K1_WARPS * 2), cap);
		k1_record_sums_g<16><<<grid, K1_THREADS, 0, st>>>(d_in, d_recs, (uint32_t)nrec, d_sums, body_from);
	} else if (avg_rec >= (12u << 10)) {
		const unsigned grid = (unsigned)std::min<size_t>((nrec + K1_WARPS * 4 - 1) / (K1_WARPS * 4), cap);
		k1_record_sums_g<8><<<grid, K1_THREADS, 0, st>>>(d_in, d_recs, (uint32_t)nrec, d_sums, body_from);
	} else {
		const unsigned grid = (unsigned)std::min<size_t>((nrec + K1_WARPS * 8 - 1) / (K1_WARPS * 8), cap);
		k1_record_sums_g<4><<<grid, K1_THREADS, 0, st>>>(d_in, d_recs, (uint32_t)nrec, d_sums, body_from);
	}
}

// K1 over a batch: per-record Fletcher-4 sums into d_sums[0..nrec)
static int32_t launch_k1(mtz_handle *h, cudaStream_t st, const uint8_t *d_in,
    const mtz_rec *d_recs, size_t nrec, RecSums *d_sums, cudaEvent_t ea, cudaEvent_t eb,
    size_t avg_rec = (128u << 10))
{
	if (nrec == 0) return MTZ_OK;
	if (ea) MTZ_CU(h, cudaEventRecord(ea, st));
	launch_k1_kernel(h, st, d_in, d_recs, nrec, d_sums, 280u, avg_rec);
	MTZ_CU(h, cudaGetLastError());
	if (eb) MTZ_CU(h, cudaEventRecord(eb, st));
	count_launch(h, 1);
	return MTZ_OK;
}

// Segmented scan of a batch's per-record sums.  phase 0: aggregate only;
// phase 1: also verify against the running checksum in h->d_carry_in.
static int32_t launch_scan(mtz_handle *h, cudaStream_t st, const RecSums *d_sums, size_t nrec,
    Part *d_tiles, ScanResult *d_res, int phase, const Ck4 *d_carry_in = nullptr)
{
	if (d_carry_in == nullptr) d_carry_in = h->d_carry_in;
	MTZ_CU(h, cudaMemsetAsync(d_res, 0, sizeof(ScanResult), st));
	if (nrec == 0) {
		MTZ_CU(h, cudaMemsetAsync(&d_res->bad, 0xff, sizeof(uint32_t), st));
		MTZ_CU(h, cudaMemcpyAsync(&d_res->carry, d_carry_in, sizeof(Ck4), cudaMemcpyDeviceToDevice, st));
		return MTZ_OK;
	}
	const unsigned ntiles = (unsigned)((nrec + SCAN_TILE - 1) / SCAN_TILE);
	k_scan_tiles<<<ntiles, SCAN_THREADS, 0, st>>>(d_sums, (uint32_t)nrec, d_tiles);
	k_scan_spine<<<1, SCAN_THREADS, 0, st>>>(d_tiles, ntiles, d_res);
	if (phase == 1)
		k_scan_verify<<<ntiles, SCAN_THREADS, 0, st>>>(d_sums, (uint32_t)nrec, d_tiles,
		    d_carry_in, d_res);
	MTZ_CU(h, cudaGetLastError());
	count_launch(h, phase == 1 ? 3 : 2);
	return MTZ_OK;
}

// ------------------------------------------------- block checksums (drr_key) --
static bool block_on(const mtz_handle *h) { return (h->cfg.flags & MTZ_FLAG_BLOCK_CKSUM) != 0; }
static bool block_sha256_on(const mtz_handle *h) { return (h->cfg.flags & MTZ_FLAG_BLOCK_SHA256) != 0; }
static bool block_sha512_on(const mtz_handle *h) { return (h->cfg.flags & MTZ_FLAG_BLOCK_SHA512) != 0; }
// VERIFY with MTZ_FLAG_BLOCK_FRAMES or MTZ_FLAG_BLOCK_LZJB: the block check encodes frames
// (kernels_frames.cuh); the other modes accept the flags and encode none
static bool block_frames_on(const mtz_handle *h)
{
	return (h->cfg.flags & (MTZ_FLAG_BLOCK_FRAMES | MTZ_FLAG_BLOCK_LZJB)) != 0 && h->cfg.mode == MTZ_MODE_VERIFY;
}
static bool block_lzjb_on(const mtz_handle *h) { return (h->cfg.flags & MTZ_FLAG_BLOCK_LZJB) != 0; }
static bool is_codec_mode(uint32_t m);
static bool cin_on(const mtz_handle *h);
static bool gzip_on(const mtz_handle *h);
static bool gzwire_on(const mtz_handle *h);
// COMPRESS / DECOMPRESS / RECOMPRESS with MTZ_FLAG_BLOCK_LOGICAL: the block check runs jobs over the
// logical bytes (launch_block_logical); VERIFY accepts the flag and does not change
static bool block_logical_on(const mtz_handle *h)
{
	return (h->cfg.flags & MTZ_FLAG_BLOCK_LOGICAL) != 0 && is_codec_mode(h->cfg.mode);
}
// block_classify's BLK_FR_* bits: LZ4 frames in VERIFY with MTZ_FLAG_BLOCK_FRAMES (the codec modes have
// their own), lzjb / zle keys with MTZ_FLAG_BLOCK_LZJB (block_classify limits them to VERIFY and RECOMPRESS,
// and to the rows of MTZ_FLAG_BLOCK_LOGICAL)
static uint32_t block_fcodecs(const mtz_handle *h)
{
	return ((h->cfg.flags & MTZ_FLAG_BLOCK_FRAMES) && h->cfg.mode == MTZ_MODE_VERIFY ? BLK_FR_LZ4 : 0u) |
	    (block_lzjb_on(h) ? BLK_FR_LZJB : 0u) | (block_logical_on(h) ? BLK_FR_LOGICAL : 0u) |
	    (cin_on(h) ? BLK_FR_CIN : 0u) | (gzip_on(h) || gzwire_on(h) ? BLK_FR_GZIP : 0u);
}
static uint32_t block_hashed(const mtz_handle *h)
{
	return (block_sha256_on(h) ? 1u << ZIO_CKSUM_SHA256 : 0u) | (block_sha512_on(h) ? 1u << ZIO_CKSUM_SHA512 : 0u);
}

static int32_t block_reset(mtz_handle *h, cudaStream_t st, BlockResult *bres)
{
	MTZ_CU(h, cudaMemsetAsync(bres, 0, offsetof(BlockResult, first_bad), st));
	MTZ_CU(h, cudaMemsetAsync(&bres->first_bad, 0xff, sizeof(BlockResult) - offsetof(BlockResult, first_bad), st));
	return MTZ_OK;
}

// k_block_check over records [0, nrec) of a (sub-)batch, record 0 being stream record `base`, then
// with MTZ_FLAG_BLOCK_SHA256 k_block_sha256 and with MTZ_FLAG_BLOCK_SHA512 k_block_sha512 over the
// same records (`d_out` = the output batch the offsets of `orecs` refer to; null with `orecs`).
// `fjobs` / `fsums`: the check's own jobs and the sums of their bytes (launch_block_frames,
// launch_block_logical).  Not counted in mtz_stats.kernel_launches: the flags leave every mtz_stats
// field as it is.
static int32_t launch_block(mtz_handle *h, cudaStream_t st, const uint8_t *d_in, const mtz_rec *d_recs,
    const RecSums *isums, const mtz_rec *orecs, const RecSums *osums, const uint8_t *d_out, size_t nrec,
    uint64_t base, BlockResult *bres, const mtz_job *fjobs = nullptr, const RecSums *fsums = nullptr)
{
	if (nrec == 0) return MTZ_OK;
	const bool sha = block_sha256_on(h), sha512 = block_sha512_on(h);
	const unsigned grid = (unsigned)((nrec + BLK_THREADS - 1) / BLK_THREADS);
	k_block_check<<<grid, BLK_THREADS, 0, st>>>(d_in, d_recs, isums, orecs, osums, d_out, (uint32_t)nrec,
	    h->cfg.mode, base, bres, block_hashed(h), fjobs, fsums, block_fcodecs(h));
	MTZ_CU(h, cudaGetLastError());
	if (sha) {
		const unsigned gs = (unsigned)((nrec + SHA_THREADS - 1) / SHA_THREADS);
		k_block_sha256<<<gs, SHA_THREADS, 0, st>>>(d_in, d_recs, d_out, orecs, (uint32_t)nrec, h->cfg.mode,
		    base, bres, fjobs, block_fcodecs(h));
		MTZ_CU(h, cudaGetLastError());
	}
	if (sha512) {
		const unsigned gs = (unsigned)((nrec + SHA512_THREADS - 1) / SHA512_THREADS);
		k_block_sha512<<<gs, SHA512_THREADS, 0, st>>>(d_in, d_recs, d_out, orecs, (uint32_t)nrec, h->cfg.mode,
		    base, bres, fjobs, block_fcodecs(h));
		MTZ_CU(h, cudaGetLastError());
	}
	return MTZ_OK;
}

static int32_t launch_k3(mtz_handle *h, cudaStream_t st, const void *d_src, void *d_dst,
    mtz_job *d_jobs, uint32_t njobs, bool compact, const uint32_t *skip = nullptr, bool count = true);
static int32_t launch_k3h(mtz_handle *h, cudaStream_t st, const void *d_src, void *d_dst,
    mtz_job *d_jobs, uint32_t njobs, uint32_t *tabs);

// The block check of a VERIFY (sub-)batch with MTZ_FLAG_BLOCK_FRAMES and/or MTZ_FLAG_BLOCK_LZJB: plan,
// K3 (LZ4 jobs, with BLOCK_FRAMES), k_lzjb_encode and k_zle_encode (lzjb / zle jobs, with BLOCK_LZJB)
// and the frame sums into cb's jobs / scratch / osums (kernels_frames.cuh), then launch_block against
// those frames.  The
// headers of records [0, nrec) lie at d_in + rec.off with rec.off - base_off < cb.scratch_cap
// (base_off 16-aligned); `compact` as for COMPRESS (all_compact_blocks).  Like the rest of the check,
// nothing here is counted in mtz_stats.
static int32_t launch_block_frames(mtz_handle *h, cudaStream_t st, CodecBufs &cb, const uint8_t *d_in,
    const mtz_rec *d_recs, const RecSums *isums, size_t nrec, uint64_t base_off, bool compact, uint64_t base,
    BlockResult *bres)
{
	if (nrec == 0) return MTZ_OK;
	if (nrec > cb.rec_cap) return fail(h, MTZ_ENOSPC, "frame batch of %zu records exceeds %zu", nrec, cb.rec_cap);
	const uint32_t n = (uint32_t)nrec;
	const uint32_t fc = block_fcodecs(h);
	uint32_t *k3_skip = (fc & BLK_FR_LZ4) && (fc & BLK_FR_LZJB) ? cb.k3_skip : nullptr;
	k_frame_plan<<<(n + FRP_THREADS - 1) / FRP_THREADS, FRP_THREADS, 0, st>>>(d_in, d_recs, n, block_hashed(h),
	    base_off, cb.d_enc, cb.enc, fc, k3_skip);
	MTZ_CU(h, cudaGetLastError());
	if (fc & BLK_FR_LZ4) {
		const int32_t rc = launch_k3(h, st, nullptr, nullptr, cb.enc, n, compact, k3_skip, false);
		if (rc != MTZ_OK) return rc;
	}
	if (fc & BLK_FR_LZJB) {
		const unsigned gl = (unsigned)std::min<size_t>((nrec + LZJB_WARPS - 1) / LZJB_WARPS, (size_t)h->sm_count * 8);
		k_lzjb_encode<<<gl, LZJB_THREADS, 0, st>>>(cb.enc, n);
		MTZ_CU(h, cudaGetLastError());
		k_zle_encode<<<gl, LZJB_THREADS, 0, st>>>(cb.enc, n);
		MTZ_CU(h, cudaGetLastError());
	}
	const unsigned gs = (unsigned)std::min<size_t>((nrec + K1_WARPS - 1) / K1_WARPS, (size_t)h->sm_count * 16);
	k_frame_sums<<<gs, K1_THREADS, 0, st>>>(cb.enc, n, cb.osums, bres);
	MTZ_CU(h, cudaGetLastError());
	return launch_block(h, st, d_in, d_recs, isums, nullptr, nullptr, nullptr, nrec, base, bres, cb.enc, cb.osums);
}

// The jobs of the block check of a codec (sub-)batch with MTZ_FLAG_BLOCK_LOGICAL, into cb.chk /
// cb.chk_sums (kernels_frames.cuh): plan, with MTZ_FLAG_BLOCK_LZJB the lzjb and zle encoders into cb.d_chk,
// and the sums of the frames and of the logical bytes of the identity jobs.  It reads the input
// batch, K2's jobs and cb.d_logical, so it runs where codec_launch_post does, after k_assemble has
// read the same; like the rest of the check, nothing here is counted in mtz_stats.
static int32_t launch_block_logical(mtz_handle *h, cudaStream_t st, CodecBufs &cb, const uint8_t *d_in,
    const mtz_rec *d_recs, size_t nrec, BlockResult *bres)
{
	const uint32_t n = (uint32_t)nrec;
	if (cb.d_chk != nullptr) MTZ_CU(h, cudaMemsetAsync(cb.chk_pos, 0, sizeof(unsigned long long), st));
	k_logical_plan<<<(n + FRP_THREADS - 1) / FRP_THREADS, FRP_THREADS, 0, st>>>(d_in, d_recs, n, h->cfg.mode,
	    block_hashed(h), block_fcodecs(h), cb.dec, cb.d_chk, cb.chk_pos, cb.chk);
	MTZ_CU(h, cudaGetLastError());
	if (cb.d_chk != nullptr) {
		const unsigned gl = (unsigned)std::min<size_t>((nrec + LZJB_WARPS - 1) / LZJB_WARPS, (size_t)h->sm_count * 8);
		k_lzjb_encode<<<gl, LZJB_THREADS, 0, st>>>(cb.chk, n);
		MTZ_CU(h, cudaGetLastError());
		k_zle_encode<<<gl, LZJB_THREADS, 0, st>>>(cb.chk, n);
		MTZ_CU(h, cudaGetLastError());
	}
	const unsigned gs = (unsigned)std::min<size_t>((nrec + K1_WARPS - 1) / K1_WARPS, (size_t)h->sm_count * 16);
	k_frame_sums<<<gs, K1_THREADS, 0, st>>>(cb.chk, n, cb.chk_sums, bres);
	MTZ_CU(h, cudaGetLastError());
	return MTZ_OK;
}

// Merge a batch's results (host copy) into `p`; on a mismatch read drr_object / drr_offset of the
// failing record from the device copy of its header (`off` = header offset in d_in).  Synchronous,
// only on the failure path.
static int32_t block_take(mtz_handle *h, BlockPending &p, const BlockResult &r, const uint8_t *d_in,
    uint64_t off)
{
	block_add(p.r, r);
	if (r.first_bad < p.r.first_bad) {
		uint64_t w[6];      // header bytes 8..55: drr_object, drr_offset, drr_checksumtype
		MTZ_CU(h, cudaMemcpy(w, d_in + off + 8, sizeof w, cudaMemcpyDeviceToHost));
		p.r.first_bad = r.first_bad;
		p.obj = w[0]; p.off = w[2]; p.ctype = (uint8_t)w[5];
	}
	return MTZ_OK;
}

// Fold the pending block verdicts into the handle.  `stream_bad` = first record of the same
// records whose stream checksum failed (~0 none): the first failing record in stream order is the
// one reported, and a record that fails both reports its stream checksum.
static int32_t block_fold(mtz_handle *h, BlockPending &p, uint64_t stream_bad)
{
	const BlockPending q = p;
	p.clear();
	{
		std::lock_guard<std::mutex> g(h->stats_mu);
		block_add(h->bstats, q.r);
	}
	if (q.r.first_bad == ~0ull || q.r.first_bad >= stream_bad) return MTZ_OK;
	{
		std::lock_guard<std::mutex> g(h->stats_mu);
		if (q.r.first_bad < h->stats.bad_record) h->stats.bad_record = q.r.first_bad;
	}
	return fail(h, MTZ_ECKSUM, "block checksum mismatch at record %llu (object %llu, offset %llu): "
	    "the bytes differ from the block on disk%s", (unsigned long long)q.r.first_bad,
	    (unsigned long long)q.obj, (unsigned long long)q.off,
	    q.ctype == ZIO_CKSUM_SHA256 ? " (sha256 key)" : q.ctype == ZIO_CKSUM_SHA512 ? " (sha512 key)" : "");
}

static int32_t ensure_dv_sums(mtz_handle *h, size_t need, cudaStream_t st)
{
	if (need <= h->dv_sums_cap) return MTZ_OK;
	size_t ncap = std::max<size_t>(need + need / 2 + 1024, 4096);
	RecSums *n = nullptr;
	MTZ_CU(h, cudaMalloc(&n, ncap * sizeof(RecSums)));
	if (h->dv_sums != nullptr) {
		if (h->dv_nrec > 0) {
			MTZ_CU(h, cudaDeviceSynchronize());
			MTZ_CU(h, cudaMemcpy(n, h->dv_sums, h->dv_nrec * sizeof(RecSums), cudaMemcpyDeviceToDevice));
		}
		MTZ_CU(h, cudaFree(h->dv_sums));
	}
	(void)st;
	h->dv_sums = n; h->dv_sums_cap = ncap;
	if (h->dv_tiles) MTZ_CU(h, cudaFree(h->dv_tiles));
	h->dv_tiles = nullptr;
	MTZ_CU(h, cudaMalloc(&h->dv_tiles, (ncap / SCAN_TILE + 2) * sizeof(Part)));
	return MTZ_OK;
}

// ------------------------------------------------------- codec pipeline ---
static bool is_codec_mode(uint32_t m)
{
	return m == MTZ_MODE_COMPRESS || m == MTZ_MODE_DECOMPRESS || m == MTZ_MODE_RECOMPRESS;
}

// RECOMPRESS proves, where it can, that a record's input frame already is what the encoder would
// emit and passes it through (K3c, kernels_lz4.cuh); MTZ_FLAG_REENCODE_ALL (or MTZ_CERTIFY=0 in the
// environment) re-encodes every record.
static bool certify_on(const mtz_handle *h)
{
	static const bool on = [] { const char *e = getenv("MTZ_CERTIFY"); return e == nullptr || atoi(e) != 0; }();
	return on && h->cfg.mode == MTZ_MODE_RECOMPRESS && !(h->cfg.flags & MTZ_FLAG_REENCODE_ALL);
}

// COMPRESS with MTZ_FLAG_LZ4_HC encodes with K3h (kernels_lz4hc.cuh) instead of K3; the other modes
// accept the flag and do not change
static bool lz4hc_on(const mtz_handle *h)
{
	return h->cfg.mode == MTZ_MODE_COMPRESS && (h->cfg.flags & MTZ_FLAG_LZ4_HC) != 0;
}

// COMPRESS with MTZ_FLAG_COMPRESSED_IN takes `zfs send -c` streams: lzjb / zle records are decoded
// (k_lzjb_decode / k_zle_decode) and re-encoded, LZ4 records forwarded; the other modes accept the
// flag and do not change
static bool cin_on(const mtz_handle *h)
{
	return h->cfg.mode == MTZ_MODE_COMPRESS && (h->cfg.flags & MTZ_FLAG_COMPRESSED_IN) != 0;
}

// ... and with MTZ_FLAG_GZIP_IN its gzip-1 .. gzip-9 records are inflated (k_inflate) and re-encoded
static bool gzip_on(const mtz_handle *h)
{
	return cin_on(h) && (h->cfg.flags & MTZ_FLAG_GZIP_IN) != 0;
}

// MTZ_FLAG_GZIP_WIRE: COMPRESS with MTZ_FLAG_COMPRESSED_IN forwards its gzip-1 .. gzip-9 records, and
// DECOMPRESS inflates them (k_inflate over cb.dec_gz); the other modes accept the flag and do not change
static bool gzwire_on(const mtz_handle *h)
{
	return (cin_on(h) || h->cfg.mode == MTZ_MODE_DECOMPRESS) && (h->cfg.flags & MTZ_FLAG_GZIP_WIRE) != 0;
}

// COMPRESS with MTZ_FLAG_GZIP_ENCODE re-codes every LZ4 frame K3 makes as a zlib frame
// (k_deflate_from_lz4) and sends the smaller; the other modes accept the flag and do not change
static bool gzenc_on(const mtz_handle *h)
{
	return h->cfg.mode == MTZ_MODE_COMPRESS && (h->cfg.flags & MTZ_FLAG_GZIP_ENCODE) != 0;
}

// K3h's hash tables: one per warp of its persistent grid (launch_k3h)
static size_t hc_tab_bytes(const mtz_handle *h)
{
	return (size_t)h->sm_count * LZ4HC_CTAS_PER_SM * LZ4HC_WARPS * LZ4HC_TAB_BYTES;
}

static int32_t codec_alloc(mtz_handle *h, CodecBufs &cb, size_t rec_cap, size_t scratch_cap)
{
	cb.rec_cap = rec_cap; cb.scratch_cap = scratch_cap;
	MTZ_CU(h, cudaMalloc(&cb.cr, rec_cap * sizeof(CodecRec)));
	MTZ_CU(h, cudaMalloc(&cb.vals, rec_cap * sizeof(uint64_t)));
	MTZ_CU(h, cudaMalloc(&cb.offs, rec_cap * sizeof(uint64_t)));
	MTZ_CU(h, cudaMalloc(&cb.out_offs, rec_cap * sizeof(uint64_t)));
	MTZ_CU(h, cudaMalloc(&cb.dec, rec_cap * sizeof(mtz_job)));
	if (gzwire_on(h) && h->cfg.mode == MTZ_MODE_DECOMPRESS) MTZ_CU(h, cudaMalloc(&cb.dec_gz, rec_cap * sizeof(mtz_job)));
	MTZ_CU(h, cudaMalloc(&cb.enc, rec_cap * sizeof(mtz_job)));
	MTZ_CU(h, cudaMalloc(&cb.out_recs, rec_cap * sizeof(mtz_rec)));
	MTZ_CU(h, cudaMalloc(&cb.osums, rec_cap * sizeof(RecSums)));
	MTZ_CU(h, cudaMalloc(&cb.steps, rec_cap * sizeof(StampStep)));
	if (h->cfg.mode == MTZ_MODE_DECOMPRESS || h->cfg.mode == MTZ_MODE_RECOMPRESS || cin_on(h))
		MTZ_CU(h, cudaMalloc(&cb.d_logical, scratch_cap + 512));
	if (h->cfg.mode != MTZ_MODE_DECOMPRESS) MTZ_CU(h, cudaMalloc(&cb.d_enc, scratch_cap + 512));
	if (gzenc_on(h)) {
		MTZ_CU(h, cudaMalloc(&cb.gz, rec_cap * sizeof(mtz_job)));
		MTZ_CU(h, cudaMalloc(&cb.d_gz, scratch_cap + 512));
	}
	if (h->cfg.mode == MTZ_MODE_VERIFY && block_lzjb_on(h) && (h->cfg.flags & MTZ_FLAG_BLOCK_FRAMES))
		MTZ_CU(h, cudaMalloc(&cb.k3_skip, rec_cap * sizeof(uint32_t)));
	if (lz4hc_on(h)) MTZ_CU(h, cudaMalloc(&cb.hc_tab, hc_tab_bytes(h)));
	if (block_logical_on(h)) {
		MTZ_CU(h, cudaMalloc(&cb.chk, rec_cap * sizeof(mtz_job)));
		MTZ_CU(h, cudaMalloc(&cb.chk_sums, rec_cap * sizeof(RecSums)));
		if (block_lzjb_on(h)) {
			MTZ_CU(h, cudaMalloc(&cb.d_chk, scratch_cap + 512));
			MTZ_CU(h, cudaMalloc(&cb.chk_pos, sizeof(unsigned long long)));
		}
	}
	if (certify_on(h)) {
		MTZ_CU(h, cudaMalloc(&cb.seq_n, rec_cap * sizeof(uint32_t)));
		MTZ_CU(h, cudaMalloc(&cb.cert, rec_cap * sizeof(uint32_t)));
	}
	MTZ_CU(h, cudaMalloc(&cb.d_cres, sizeof(CodecResult)));
	MTZ_CU(h, cudaHostAlloc(&cb.h_cres, sizeof(CodecResult), cudaHostAllocDefault));
	MTZ_CU(h, cudaMalloc(&cb.d_ores, sizeof(ScanResult)));
	MTZ_CU(h, cudaHostAlloc(&cb.h_ores, sizeof(ScanResult), cudaHostAllocDefault));
	MTZ_CU(h, cudaMalloc(&cb.d_outpos, sizeof(uint64_t)));
	MTZ_CU(h, cudaMemset(cb.d_outpos, 0, sizeof(uint64_t)));
	return MTZ_OK;
}

static void codec_free(CodecBufs &cb)
{
	cudaFree(cb.cr); cudaFree(cb.vals); cudaFree(cb.offs); cudaFree(cb.out_offs);
	cudaFree(cb.dec); cudaFree(cb.dec_gz); cudaFree(cb.enc); cudaFree(cb.out_recs); cudaFree(cb.osums); cudaFree(cb.steps);
	cudaFree(cb.d_logical); cudaFree(cb.d_enc); cudaFree(cb.d_cres); cudaFree(cb.d_ores);
	cudaFree(cb.d_outpos); cudaFree(cb.seq_n); cudaFree(cb.cert); cudaFree(cb.k3_skip); cudaFree(cb.hc_tab);
	cudaFree(cb.chk); cudaFree(cb.chk_sums); cudaFree(cb.d_chk); cudaFree(cb.chk_pos);
	cudaFree(cb.gz); cudaFree(cb.d_gz);
	if (cb.h_cres) cudaFreeHost(cb.h_cres);
	if (cb.h_ores) cudaFreeHost(cb.h_ores);
	cb = CodecBufs();
}

// start of a codec batch: output offset 0, no bad record, counters zero
static int32_t codec_reset(mtz_handle *h, cudaStream_t st, CodecBufs &cb)
{
	MTZ_CU(h, cudaMemsetAsync(cb.d_outpos, 0, sizeof(uint64_t), st));
	MTZ_CU(h, cudaMemsetAsync(cb.d_cres, 0, sizeof(CodecResult), st));
	MTZ_CU(h, cudaMemsetAsync(&cb.d_cres->bad, 0xff, sizeof(uint32_t), st));
	MTZ_CU(h, cudaMemsetAsync(cb.d_ores, 0, sizeof(ScanResult), st));
	return MTZ_OK;
}

// Part 1 of the re-encoding pipeline of one (sub-)batch: plan + K2 + K3.  It
// does not touch the running checksums, so it may run ahead of the chain.
static int32_t launch_k3c(mtz_handle *h, cudaStream_t st, CodecBufs &cb, uint32_t njobs, bool compact);

// true when every DRR_WRITE of the table has a 128 KiB-class logical size
static bool all_compact_blocks(const mtz_rec *recs, size_t n)
{
	for (size_t i = 0; i < n; i++)
		if (recs[i].type == 3 && (recs[i].lsize < (uint32_t)LZ4_64KLIMIT || recs[i].lsize > 131072u))
			return false;
	return true;
}

static int32_t codec_launch_dec(mtz_handle *h, cudaStream_t st, CodecBufs &cb, const uint8_t *d_in,
    const mtz_rec *d_recs, size_t nrec);
static int32_t codec_launch_enc(mtz_handle *h, cudaStream_t st, CodecBufs &cb, size_t nrec, bool compact,
    cudaEvent_t ka = nullptr, cudaEvent_t kb = nullptr, cudaStream_t st_k3 = nullptr);

static int32_t codec_launch_pre(mtz_handle *h, cudaStream_t st, CodecBufs &cb, const uint8_t *d_in,
    const mtz_rec *d_recs, size_t nrec, cudaEvent_t ea, cudaEvent_t eb, bool compact,
    cudaEvent_t ka = nullptr, cudaEvent_t kb = nullptr, cudaStream_t st_k3 = nullptr)
{
	if (nrec == 0) return MTZ_OK;
	if (ea) MTZ_CU(h, cudaEventRecord(ea, st));
	int32_t rc = codec_launch_dec(h, st, cb, d_in, d_recs, nrec);
	if (rc != MTZ_OK) return rc;
	rc = codec_launch_enc(h, st, cb, nrec, compact, ka, kb, st_k3);
	if (rc != MTZ_OK) return rc;
	if (eb) MTZ_CU(h, cudaEventRecord(eb, st));
	return MTZ_OK;
}

// plan + K2 (decode) of one (sub-)batch; in COMPRESS with MTZ_FLAG_COMPRESSED_IN the lzjb and zle
// decoders, and with MTZ_FLAG_GZIP_IN k_inflate, in K2's place (every decode job of that mode is one
// of theirs); in DECOMPRESS with MTZ_FLAG_GZIP_WIRE k_inflate after K2, over the gzip jobs that
// k_plan_jobs kept out of K2's table
static int32_t codec_launch_dec(mtz_handle *h, cudaStream_t st, CodecBufs &cb, const uint8_t *d_in,
    const mtz_rec *d_recs, size_t nrec)
{
	if (nrec == 0) return MTZ_OK;
	if (nrec > cb.rec_cap) return fail(h, MTZ_ENOSPC, "codec batch of %zu records exceeds %zu", nrec, cb.rec_cap);
	const uint32_t n = (uint32_t)nrec, mode = h->cfg.mode;
	const unsigned tb = 256, gb = (n + tb - 1) / tb;
	k_plan_need<<<gb, tb, 0, st>>>(d_recs, n, mode, cb.cr, cb.vals, cin_on(h), gzip_on(h), gzwire_on(h));
	k_xscan_u64<<<1, XSCAN_THREADS, 0, st>>>(cb.vals, cb.offs, n, nullptr, nullptr);
	k_plan_jobs<<<gb, tb, 0, st>>>(d_in, d_recs, n, cb.cr, cb.offs, cb.d_logical, cb.d_enc, cb.dec, cb.enc,
	    cb.dec_gz);
	MTZ_CU(h, cudaGetLastError());
	count_launch(h, 3);
	if (mode != MTZ_MODE_COMPRESS) {
		int32_t rc = launch_k2(h, st, nullptr, nullptr, cb.dec, n, cb.seq_n ? cb.enc : nullptr, cb.seq_n);
		if (rc != MTZ_OK) return rc;
		if (cb.dec_gz != nullptr) {
			const unsigned gi = (unsigned)std::min<size_t>((nrec + INFL_WARPS - 1) / INFL_WARPS, (size_t)h->sm_count * 8);
			k_inflate<<<gi, INFL_THREADS, 0, st>>>(d_recs, cb.dec_gz, n);
			MTZ_CU(h, cudaGetLastError());
			count_launch(h, 1);
		}
	} else if (cin_on(h)) {
		const unsigned gl = (unsigned)std::min<size_t>((nrec + LZJB_WARPS - 1) / LZJB_WARPS, (size_t)h->sm_count * 8);
		k_lzjb_decode<<<gl, LZJB_THREADS, 0, st>>>(d_recs, cb.dec, n);
		k_zle_decode<<<gl, LZJB_THREADS, 0, st>>>(d_recs, cb.dec, n);
		MTZ_CU(h, cudaGetLastError());
		count_launch(h, 2);
		if (gzip_on(h)) {
			const unsigned gi = (unsigned)std::min<size_t>((nrec + INFL_WARPS - 1) / INFL_WARPS, (size_t)h->sm_count * 8);
			k_inflate<<<gi, INFL_THREADS, 0, st>>>(d_recs, cb.dec, n);
			MTZ_CU(h, cudaGetLastError());
			count_launch(h, 1);
		}
	}
	return MTZ_OK;
}

// the grid of k_deflate_from_lz4 over n jobs
static unsigned defl_grid(const mtz_handle *h, size_t n)
{
	return (unsigned)std::max<size_t>(1, std::min<size_t>((n + DEFL_WARPS - 1) / DEFL_WARPS, (size_t)h->sm_count * 8));
}

// K3 (encode) of one (sub-)batch, and with MTZ_FLAG_GZIP_ENCODE the deflate re-coding of its frames
// With `st_k3` (and both events) the encoder runs on that low-priority side stream, forked from
// and joined back into `st`, so that the rest of this slot's work keeps `st`'s high priority.
static int32_t codec_launch_enc(mtz_handle *h, cudaStream_t st, CodecBufs &cb, size_t nrec, bool compact,
    cudaEvent_t ka, cudaEvent_t kb, cudaStream_t st_k3)
{
	if (nrec == 0 || h->cfg.mode == MTZ_MODE_DECOMPRESS) return MTZ_OK;
	if (st_k3 == nullptr || ka == nullptr || kb == nullptr) st_k3 = st;
	if (ka) MTZ_CU(h, cudaEventRecord(ka, st));
	if (st_k3 != st) MTZ_CU(h, cudaStreamWaitEvent(st_k3, ka, 0));
	int32_t rc = MTZ_OK;
	if (cb.hc_tab != nullptr) {
		rc = launch_k3h(h, st_k3, nullptr, nullptr, cb.enc, (uint32_t)nrec, cb.hc_tab);
	} else {
		if (cb.cert != nullptr) rc = launch_k3c(h, st_k3, cb, (uint32_t)nrec, compact);
		if (rc == MTZ_OK) rc = launch_k3(h, st_k3, nullptr, nullptr, cb.enc, (uint32_t)nrec, compact, cb.cert);
		if (rc == MTZ_OK && cb.gz != nullptr) {
			// frames at d_enc + slot are re-coded into d_gz + slot: gz_base moves a d_enc address there
			k_deflate_from_lz4<<<defl_grid(h, nrec), DEFL_THREADS, 0, st_k3>>>(cb.enc, cb.gz, (uint32_t)nrec, 0ull, 0ull,
			    (uint64_t)(uintptr_t)cb.d_gz - (uint64_t)(uintptr_t)cb.d_enc, true);
			if (cudaGetLastError() != cudaSuccess) rc = fail(h, MTZ_ECUDA, "k_deflate_from_lz4 launch");
			else count_launch(h, 1);
		}
	}
	if (rc == MTZ_OK && kb) MTZ_CU(h, cudaEventRecord(kb, st_k3));
	if (rc == MTZ_OK && st_k3 != st) MTZ_CU(h, cudaStreamWaitEvent(st, kb, 0));
	return rc;
}

// Part 2: layout, assemble into d_out + *cb.d_outpos (the running output offset
// lives on the device so sub-batches chain without a host round trip), sums of
// the output records, and the sequential stamp chain from h->d_carry_out.
// With `bres` the block check runs on the output sums as well (`isums` = the input's sums of these
// records, `bbase` = stream index of the first of them).
static int32_t codec_launch_post(mtz_handle *h, cudaStream_t st, CodecBufs &cb, const uint8_t *d_in,
    const mtz_rec *d_recs, size_t nrec, uint8_t *d_out, uint32_t rec_base,
    mtz_rec *all_orecs = nullptr, RecSums *all_osums = nullptr, Ck4 *d_carry_out = nullptr,
    const RecSums *isums = nullptr, uint64_t bbase = 0, BlockResult *bres = nullptr)
{
	if (nrec == 0) return MTZ_OK;
	if (d_carry_out == nullptr) d_carry_out = h->d_carry_out;
	// shard mode: output record table / sums are kept for the whole submit and the
	// stamp chain runs later (mtz_dev_finish) from the previous shard's checksum
	mtz_rec *orecs = all_orecs ? all_orecs + rec_base : cb.out_recs;
	RecSums *osums = all_osums ? all_osums + rec_base : cb.osums;
	const uint32_t n = (uint32_t)nrec, mode = h->cfg.mode;
	const unsigned tb = 256, gb = (n + tb - 1) / tb;
	k_layout<<<gb, tb, 0, st>>>(d_recs, n, cb.cr, cb.dec, cb.enc, cb.vals, cb.d_cres, rec_base, cb.cert, cb.dec_gz, cb.gz);
	k_xscan_u64<<<1, XSCAN_THREADS, 0, st>>>(cb.vals, cb.out_offs, n, cb.d_outpos, cb.d_outpos);
	const unsigned ga = (unsigned)std::min<size_t>((n + 7) / 8, (size_t)h->sm_count * 8);
	k_assemble<<<ga, ASM_THREADS, 0, st>>>(d_in, d_recs, n, mode, cb.cr, cb.out_offs, cb.enc,
	    cb.d_logical, cb.d_enc, d_out, orecs, cb.cert, cb.gz);
	MTZ_CU(h, cudaGetLastError());
	// output records of a codec batch are smaller than the logical size: decide by the input's
	launch_k1_kernel(h, st, d_out, orecs, n, osums, 312u, cb.avg_out_rec);
	if (bres != nullptr) {
		int32_t rc = block_logical_on(h) ? launch_block_logical(h, st, cb, d_in, d_recs, nrec, bres) : MTZ_OK;
		if (rc == MTZ_OK)
			rc = launch_block(h, st, d_in, d_recs, isums, orecs, osums, d_out, nrec, bbase, bres, cb.chk, cb.chk_sums);
		if (rc != MTZ_OK) return rc;
	}
	if (all_osums == nullptr) {
		const unsigned gp = (n + 127u) / 128u;
		k_stamp_prep<<<gp, 128, 0, st>>>(orecs, osums, n, cb.steps);
		k_stamp_chain<<<1, STAMP_THREADS, 0, st>>>(d_out, orecs, osums, cb.steps, n, d_carry_out, cb.d_ores);
		count_launch(h, 2);
	}
	MTZ_CU(h, cudaGetLastError());
	MTZ_CU(h, cudaMemcpyAsync(&cb.d_cres->out_bytes, cb.d_outpos, sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
	count_launch(h, 4);
	return MTZ_OK;
}

// ------------------------------------------------------------ device API --
int32_t mtz_dev_reset(mtz_handle *h)
{
	CHECK_H(h);
	MTZ_CU(h, cudaSetDevice(h->device));
	MTZ_CU(h, cudaMemsetAsync(h->d_carry_in, 0, sizeof(Ck4), h->st));
	MTZ_CU(h, cudaMemsetAsync(h->d_carry_out, 0, sizeof(Ck4), h->st));
	MTZ_CU(h, cudaStreamSynchronize(h->st));
	h->records_done = 0;
	h->dv_nrec = 0; h->dv_in_bytes = 0;
	h->dv_bres_live = false;
	h->bpend.clear();
	std::lock_guard<std::mutex> g(h->stats_mu);
	h->stats = mtz_stats();
	h->stats.bad_record = ~0ull;
	h->bstats = mtz_block_stats();
	if (block_on(h)) h->bstats.first_frame_miss = ~0ull;
	h->cstats = mtz_compressed_in_stats();
	return MTZ_OK;
}

int32_t mtz_set_carry(mtz_handle *h, const uint64_t carry_in[4], const uint64_t carry_out[4])
{
	CHECK_H(h);
	MTZ_CU(h, cudaSetDevice(h->device));
	if (carry_in) MTZ_CU(h, cudaMemcpy(h->d_carry_in, carry_in, 32, cudaMemcpyHostToDevice));
	if (carry_out) MTZ_CU(h, cudaMemcpy(h->d_carry_out, carry_out, 32, cudaMemcpyHostToDevice));
	return MTZ_OK;
}

// The device API's scratch.  dv_cb: the codec sub-batches, or in VERIFY the frames of the block check
// (MTZ_FLAG_BLOCK_FRAMES); the codec modes also get a second set and the streams and events of their
// three-stream pipeline.
static int32_t dv_alloc(mtz_handle *h)
{
	if (h->dv_cb.cr != nullptr) return MTZ_OK;
	const size_t scratch = std::max<size_t>(2ull << 30, (size_t)h->cfg.batch_bytes + MAX_RECORD_BYTES);
	int32_t rc = codec_alloc(h, h->dv_cb, 65536, scratch);
	if (rc != MTZ_OK || !is_codec_mode(h->cfg.mode)) return rc;
	rc = codec_alloc(h, h->dv_cb2, 65536, scratch);
	if (rc != MTZ_OK) return rc;
	// one set of results / running output offset for the whole submit
	cudaFree(h->dv_cb2.d_cres); cudaFree(h->dv_cb2.d_ores); cudaFree(h->dv_cb2.d_outpos);
	cudaFreeHost(h->dv_cb2.h_cres); cudaFreeHost(h->dv_cb2.h_ores);
	h->dv_cb2.d_cres = h->dv_cb.d_cres; h->dv_cb2.d_ores = h->dv_cb.d_ores;
	h->dv_cb2.d_outpos = h->dv_cb.d_outpos;
	h->dv_cb2.h_cres = h->dv_cb.h_cres; h->dv_cb2.h_ores = h->dv_cb.h_ores;
	MTZ_CU(h, cudaEventCreate(&h->dv_c0));
	MTZ_CU(h, cudaEventCreate(&h->dv_c1));
	MTZ_CU(h, make_stream(&h->st_post, true));
	MTZ_CU(h, make_stream(&h->st_dec, true));
	for (int i = 0; i < 2; i++) {
		MTZ_CU(h, cudaEventCreateWithFlags(&h->ev_dec[i], cudaEventDisableTiming));
		MTZ_CU(h, cudaEventCreateWithFlags(&h->ev_pre[i], cudaEventDisableTiming));
		if (i == 0) MTZ_CU(h, cudaEventCreateWithFlags(&h->ev_reset, cudaEventDisableTiming));
		MTZ_CU(h, cudaEventCreateWithFlags(&h->ev_post[i], cudaEventDisableTiming));
	}
	return MTZ_OK;
}

// host copy of the submit's record table (dv_hrecs): the sub-batches are cut on the host
static int32_t dv_host_recs(mtz_handle *h, cudaStream_t st, const mtz_rec *d_recs, size_t nrec)
{
	h->dv_hrecs.resize(nrec);
	MTZ_CU(h, cudaMemcpyAsync(h->dv_hrecs.data(), d_recs, nrec * sizeof(mtz_rec), cudaMemcpyDeviceToHost, st));
	MTZ_CU(h, cudaStreamSynchronize(st));
	return MTZ_OK;
}

// The block check of a VERIFY submit with MTZ_FLAG_BLOCK_FRAMES / _LZJB, in sub-batches whose input span fits
// dv_cb's scratch (2 GiB) and whose records fit its tables; one after another on `st`, verdicts into
// dv_bres for the finish.
static int32_t dv_block_frames(mtz_handle *h, cudaStream_t st, const uint8_t *d_in, const mtz_rec *d_recs,
    size_t nrec)
{
	int32_t rc = dv_alloc(h);
	if (rc == MTZ_OK) rc = dv_host_recs(h, st, d_recs, nrec);
	if (rc != MTZ_OK) return rc;
	const CodecBufs &cb = h->dv_cb;
	const mtz_rec *hr = h->dv_hrecs.data();
	for (size_t i0 = 0; i0 < nrec;) {
		const uint64_t base_off = hr[i0].off & ~15ull;
		size_t i1 = i0;
		while (i1 < nrec && i1 - i0 < cb.rec_cap) {
			const uint64_t end = hr[i1].off + DRR_HDR + hr[i1].payload;
			if (end - base_off > cb.scratch_cap) {
				if (i1 == i0) return fail(h, MTZ_ENOSPC, "record exceeds the frame scratch");
				break;
			}
			i1++;
		}
		rc = launch_block_frames(h, st, h->dv_cb, d_in, d_recs + i0, h->dv_sums + i0, i1 - i0, base_off,
		    all_compact_blocks(hr + i0, i1 - i0), h->dv_first + i0, h->dv_bres);
		if (rc != MTZ_OK) return rc;
		i0 = i1;
	}
	return MTZ_OK;
}

int32_t mtz_dev_submit(mtz_handle *h, const void *d_in, size_t in_bytes,
    const mtz_rec *d_recs, size_t nrec, void *d_out, size_t out_cap, void *cuda_stream)
{
	CHECK_H(h);
	(void)d_out; (void)out_cap;
	if (nrec > 0xfffffff0ull) return fail(h, MTZ_EINVAL, "too many records in one batch");
	if (((uintptr_t)d_in & 3) != 0) return fail(h, MTZ_EINVAL, "d_in must be 4-byte aligned");
	if (h->cfg.mode == MTZ_MODE_PASSTHROUGH)
		return fail(h, MTZ_EINVAL, "mtz_dev_submit: no device path for PASSTHROUGH");
	MTZ_CU(h, cudaSetDevice(h->device));
	cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : h->st;
	int32_t rc = ensure_dv_sums(h, nrec, st);
	if (rc != MTZ_OK) return rc;
	h->dv_nrec = nrec; h->dv_in_bytes = in_bytes; h->dv_st = st;
	h->dv_first = h->records_done;
	rc = launch_k1(h, st, (const uint8_t *)d_in, d_recs, nrec, h->dv_sums, h->dv_k1a, h->dv_k1b,
	    nrec ? in_bytes / nrec : 0);
	h->dv_timed = (rc == MTZ_OK && nrec > 0);
	if (rc != MTZ_OK) return rc;
	h->dv_bres_live = block_on(h) && nrec > 0;
	if (h->dv_bres_live) {
		h->dv_in = (const uint8_t *)d_in; h->dv_recs = d_recs;
		rc = block_reset(h, st, h->dv_bres);
		if (rc == MTZ_OK && block_frames_on(h))
			rc = dv_block_frames(h, st, (const uint8_t *)d_in, d_recs, nrec);
		else if (rc == MTZ_OK && !is_codec_mode(h->cfg.mode))
			rc = launch_block(h, st, (const uint8_t *)d_in, d_recs, h->dv_sums, nullptr, nullptr, nullptr,
			    nrec, h->dv_first, h->dv_bres);
		if (rc != MTZ_OK) return rc;
	}
	if (!is_codec_mode(h->cfg.mode)) return MTZ_OK;

	// ---- re-encoding modes: bounded-scratch sub-batches, output chained on device.
	// Two scratch sets and a second stream: plan+K2+K3 of sub-batch k+1 (stream st)
	// overlap layout/assemble/sums/stamp-chain of sub-batch k (stream st_post); the
	// chain is one warp on one SM and would otherwise serialise ~12 % of the step.
	if (d_out == nullptr) return fail(h, MTZ_EINVAL, "codec modes need d_out");
	rc = dv_alloc(h);
	if (rc != MTZ_OK) return rc;
	rc = dv_host_recs(h, st, d_recs, nrec);
	if (rc != MTZ_OK) return rc;
	rc = codec_reset(h, st, h->dv_cb);
	if (rc != MTZ_OK) return rc;
	size_t need_out = 0;
	for (size_t i = 0; i < nrec; i++)
		need_out += DRR_HDR + std::max<size_t>(h->dv_hrecs[i].payload,
		    h->dv_hrecs[i].type == 3 ? h->dv_hrecs[i].lsize : 0);
	if (need_out > out_cap)
		return fail(h, MTZ_ENOSPC, "d_out must hold the worst case of %zu bytes", need_out);
	const bool defer = (h->cfg.flags & MTZ_FLAG_DEFER_VERIFY) != 0;
	if (defer && nrec > h->dv_all_cap) {
		if (h->dv_all_orecs) MTZ_CU(h, cudaFree(h->dv_all_orecs));
		if (h->dv_all_osums) MTZ_CU(h, cudaFree(h->dv_all_osums));
		if (h->dv_all_steps) MTZ_CU(h, cudaFree(h->dv_all_steps));
		h->dv_all_orecs = nullptr; h->dv_all_osums = nullptr; h->dv_all_steps = nullptr;
		h->dv_all_cap = nrec + nrec / 8 + 64;
		MTZ_CU(h, cudaMalloc(&h->dv_all_orecs, h->dv_all_cap * sizeof(mtz_rec)));
		MTZ_CU(h, cudaMalloc(&h->dv_all_osums, h->dv_all_cap * sizeof(RecSums)));
		MTZ_CU(h, cudaMalloc(&h->dv_all_steps, h->dv_all_cap * sizeof(StampStep)));
	}
	h->dv_out = (uint8_t *)d_out;
	MTZ_CU(h, cudaEventRecord(h->dv_c0, st));
	// codec_reset (and whatever this stream did before) is ordered before anything the decode
	// and post streams do for this submit.  A dedicated event: ev_pre[0] is re-recorded after
	// K3 of sub-batch 0, so waiting on it here would make K2 of sub-batch 1 wait for that K3
	// instead of running under it.
	MTZ_CU(h, cudaEventRecord(h->ev_reset, st));
	MTZ_CU(h, cudaStreamWaitEvent(h->st_post, h->ev_reset, 0));
	bool used[2] = { false, false };
	size_t k = 0;
	for (size_t i0 = 0; i0 < nrec; k++) {
		size_t i1 = i0, budget = 0;
		CodecBufs &cb = (k & 1) ? h->dv_cb2 : h->dv_cb;
		while (i1 < nrec && (i1 - i0) < cb.rec_cap) {
			const mtz_rec &r = h->dv_hrecs[i1];
			const size_t cost = std::max<size_t>(r.payload, r.type == 3 ? r.lsize : 0) + 64;
			if (cost > cb.scratch_cap) return fail(h, MTZ_ENOSPC, "record exceeds the codec scratch");
			if (i1 > i0 && budget + cost > cb.scratch_cap) break;
			budget += cost; i1++;
		}
		const int b = (int)(k & 1);
		// decode stream: plan + K2 of sub-batch k run under K3 of sub-batch k-1 (K2 needs no
		// shared memory and K3 leaves 40 warp slots per SM empty)
		if (used[b]) MTZ_CU(h, cudaStreamWaitEvent(h->st_dec, h->ev_post[b], 0));   // scratch set free again
		else MTZ_CU(h, cudaStreamWaitEvent(h->st_dec, h->ev_reset, 0));            // after codec_reset
		rc = codec_launch_dec(h, h->st_dec, cb, (const uint8_t *)d_in, d_recs + i0, i1 - i0);
		if (rc != MTZ_OK) return rc;
		MTZ_CU(h, cudaEventRecord(h->ev_dec[b], h->st_dec));
		MTZ_CU(h, cudaStreamWaitEvent(st, h->ev_dec[b], 0));
		while (h->dv_k3ev.size() < 2 * (k + 1)) {
			cudaEvent_t ev = nullptr;
			MTZ_CU(h, cudaEventCreate(&ev));
			h->dv_k3ev.push_back(ev);
		}
		rc = codec_launch_enc(h, st, cb, i1 - i0, all_compact_blocks(h->dv_hrecs.data() + i0, i1 - i0),
		    h->cfg.mode == MTZ_MODE_DECOMPRESS ? nullptr : h->dv_k3ev[2 * k],
		    h->cfg.mode == MTZ_MODE_DECOMPRESS ? nullptr : h->dv_k3ev[2 * k + 1]);
		if (rc != MTZ_OK) return rc;
		MTZ_CU(h, cudaEventRecord(h->ev_pre[b], st));
		MTZ_CU(h, cudaStreamWaitEvent(h->st_post, h->ev_pre[b], 0));
		rc = codec_launch_post(h, h->st_post, cb, (const uint8_t *)d_in, d_recs + i0, i1 - i0,
		    (uint8_t *)d_out, (uint32_t)i0, defer ? h->dv_all_orecs : nullptr,
		    defer ? h->dv_all_osums : nullptr, nullptr, h->dv_sums + i0, h->dv_first + i0,
		    h->dv_bres_live ? h->dv_bres : nullptr);
		if (rc != MTZ_OK) return rc;
		MTZ_CU(h, cudaEventRecord(h->ev_post[b], h->st_post));
		used[b] = true;
		i0 = i1;
	}
	for (int b = 0; b < 2; b++)
		if (used[b]) MTZ_CU(h, cudaStreamWaitEvent(st, h->ev_post[b], 0));
	MTZ_CU(h, cudaEventRecord(h->dv_c1, st));
	h->dv_k3n = (h->cfg.mode == MTZ_MODE_DECOMPRESS) ? 0 : k;
	return MTZ_OK;
}

int32_t mtz_dev_aggregate(mtz_handle *h, uint64_t agg[5])
{
	CHECK_H(h);
	if (agg == nullptr) return MTZ_EINVAL;
	MTZ_CU(h, cudaSetDevice(h->device));
	cudaStream_t st = h->dv_st ? h->dv_st : h->st;
	int32_t rc = launch_scan(h, st, h->dv_sums, h->dv_nrec, h->dv_tiles, h->dv_res, 0);
	if (rc != MTZ_OK) return rc;
	MTZ_CU(h, cudaMemcpyAsync(h->dv_hres, h->dv_res, sizeof(ScanResult), cudaMemcpyDeviceToHost, st));
	MTZ_CU(h, cudaStreamSynchronize(st));
	agg[0] = h->dv_hres->agg.n; agg[1] = h->dv_hres->agg.a; agg[2] = h->dv_hres->agg.b;
	agg[3] = h->dv_hres->agg.c; agg[4] = h->dv_hres->agg.d;
	return MTZ_OK;
}

// `bp`: block-check verdicts of the same records (MTZ_FLAG_BLOCK_CKSUM), folded in with them
static int32_t account_result(mtz_handle *h, const ScanResult &r, uint64_t first_rec, size_t nrec,
    size_t bytes_in, size_t bytes_out, BlockPending *bp = nullptr)
{
	{
		std::lock_guard<std::mutex> g(h->stats_mu);
		h->stats.batches += 1;
		h->stats.records += nrec;
		h->stats.bytes_in += bytes_in;
		h->stats.bytes_out += bytes_out;
		if (r.end_seen) {
			h->stats.end_seen = 1;
			memcpy(h->end_ck, &r.end_ck, 32);
		}
	}
	if (bp != nullptr) {
		const int32_t rc = block_fold(h, *bp, r.bad != 0xffffffffu ? first_rec + r.bad : ~0ull);
		if (rc != MTZ_OK) return rc;
	}
	if (r.bad != 0xffffffffu) {
		const uint64_t bad = first_rec + r.bad;
		{
			std::lock_guard<std::mutex> g(h->stats_mu);
			if (bad < h->stats.bad_record) h->stats.bad_record = bad;
		}
		return fail(h, MTZ_ECKSUM, "stream checksum mismatch at record %llu",
		    (unsigned long long)bad);
	}
	return MTZ_OK;
}

int32_t mtz_dev_aggregate_async(mtz_handle *h, void *d_agg)
{
	CHECK_H(h);
	if (d_agg == nullptr) return MTZ_EINVAL;
	MTZ_CU(h, cudaSetDevice(h->device));
	cudaStream_t st = h->dv_st ? h->dv_st : h->st;
	int32_t rc = launch_scan(h, st, h->dv_sums, h->dv_nrec, h->dv_tiles, h->dv_res, 0);
	if (rc != MTZ_OK) return rc;
	MTZ_CU(h, cudaMemcpyAsync(d_agg, &h->dv_res->agg, sizeof(Part), cudaMemcpyDeviceToDevice, st));
	return MTZ_OK;
}

static int32_t dev_finish_impl(mtz_handle *h, const uint64_t carry_in[4], const void *d_all_aggs,
    uint32_t rank, const uint64_t carry_out_in[4], size_t *out_bytes, uint64_t carry[4],
    uint64_t carry_out[4], bool xchg = false);

int32_t mtz_dev_finish(mtz_handle *h, const uint64_t carry_in[4], const uint64_t carry_out_in[4],
    size_t *out_bytes, uint64_t carry[4], uint64_t carry_out[4])
{
	return dev_finish_impl(h, carry_in, nullptr, 0, carry_out_in, out_bytes, carry, carry_out);
}

int32_t mtz_dev_finish_gathered(mtz_handle *h, const void *d_all_aggs, uint32_t rank,
    const uint64_t carry_out_in[4], size_t *out_bytes, uint64_t carry[4], uint64_t carry_out[4])
{
	if (d_all_aggs == nullptr) return MTZ_EINVAL;
	return dev_finish_impl(h, nullptr, d_all_aggs, rank, carry_out_in, out_bytes, carry, carry_out);
}

// ---- library-owned NCCL for the one-process-per-GPU shard form -----------------------------
int32_t mtz_comm_unique_id(uint8_t id[128])
{
	if (id == nullptr) return MTZ_EINVAL;
	static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
	ncclUniqueId u;
	if (!nccl_available(nullptr)) return MTZ_ECUDA;
	if (ncclGetUniqueId(&u) != ncclSuccess) return MTZ_ECUDA;
	memcpy(id, &u, 128);
	return MTZ_OK;
}

int32_t mtz_comm_init(mtz_handle *h, const uint8_t id[128], int32_t rank, int32_t world)
{
	CHECK_H(h);
	if (id == nullptr || world < 1 || rank < 0 || rank >= world) return fail(h, MTZ_EINVAL, "bad rank/world");
	if (h->xcomm != nullptr) return fail(h, MTZ_EINVAL, "communicator already initialised");
	std::string why;
	if (!nccl_available(&why)) return fail(h, MTZ_ECUDA, "the shard exchange needs NCCL: %s", why.c_str());
	MTZ_CU(h, cudaSetDevice(h->device));
	ncclUniqueId u;
	memcpy(&u, id, 128);
	MTZ_NCCL(h, ncclCommInitRank(&h->xcomm, world, u, rank));
	h->xcomm_owned = true;
	h->xrank = rank; h->xworld = world;
	MTZ_CU(h, cudaMalloc(&h->d_xagg, sizeof(Part)));
	MTZ_CU(h, cudaMalloc(&h->d_xall, (size_t)world * sizeof(Part)));
	MTZ_CU(h, cudaMalloc(&h->d_xbase, 2 * sizeof(Ck4)));
	return MTZ_OK;
}

int32_t mtz_comm_share(mtz_handle *h, mtz_handle *owner)
{
	CHECK_H(h);
	if (owner == nullptr || owner->xcomm == nullptr) return fail(h, MTZ_EINVAL, "the owner has no communicator");
	if (h->xcomm != nullptr) return fail(h, MTZ_EINVAL, "communicator already initialised");
	if (h->device != owner->device) return fail(h, MTZ_EINVAL, "a shared communicator needs the same device");
	MTZ_CU(h, cudaSetDevice(h->device));
	h->xcomm = owner->xcomm; h->xcomm_owned = false;
	h->xrank = owner->xrank; h->xworld = owner->xworld;
	MTZ_CU(h, cudaMalloc(&h->d_xagg, sizeof(Part)));
	MTZ_CU(h, cudaMalloc(&h->d_xall, (size_t)h->xworld * sizeof(Part)));
	MTZ_CU(h, cudaMalloc(&h->d_xbase, 2 * sizeof(Ck4)));
	return MTZ_OK;
}

int32_t mtz_dev_finish_exchange(mtz_handle *h, const uint64_t round_base_in[4], uint32_t flags,
    size_t *out_bytes, uint64_t carry[4], uint64_t carry_out[4], uint64_t round_base_out[4])
{
	CHECK_H(h);
	if (h->xcomm == nullptr) return fail(h, MTZ_EINVAL, "mtz_comm_init first");
	MTZ_CU(h, cudaSetDevice(h->device));
	cudaStream_t st = h->dv_st ? h->dv_st : h->st;
	h->xflags = flags;
	if (round_base_in != nullptr) {
		memcpy(&h->h_carry[2], round_base_in, 32);
		MTZ_CU(h, cudaMemcpyAsync(&h->d_xbase[0], &h->h_carry[2], 32, cudaMemcpyHostToDevice, st));
	} else {
		MTZ_CU(h, cudaMemsetAsync(&h->d_xbase[0], 0, 32, st));
	}
	// The output checksum arrives from the rank that holds the chunk before this one.  Communicator
	// operations execute in issue order, so every rank must issue them in an order compatible with
	//   AG_0 | S_0 R_1 | S_1 R_2 | ... | S_N-1 R_N | AG_1 | S_N R_N+1 | ...
	// (chunk j on rank j % N, AG_k the all-gather of round k): rank 0 receives the END of the
	// previous round BEFORE this round's all-gather, every other rank after it -- any other
	// placement makes the all-gather and a send wait for each other.
	const bool hop = is_codec_mode(h->cfg.mode) && (h->cfg.flags & MTZ_FLAG_DEFER_VERIFY) && !(flags & MTZ_XCHG_FIRST);
	const int from = (h->xrank + h->xworld - 1) % h->xworld;
	if (hop && h->xrank == 0)
		MTZ_NCCL(h, ncclRecv(h->d_carry_out, 4, ncclUint64, from, h->xcomm, st));
	// the 40-byte aggregate of this chunk -> all ranks (the path's one collective, SURVEY 8e)
	int32_t rc = launch_scan(h, st, h->dv_sums, h->dv_nrec, h->dv_tiles, h->dv_res, 0);
	if (rc != MTZ_OK) return rc;
	MTZ_CU(h, cudaMemcpyAsync(h->d_xagg, &h->dv_res->agg, sizeof(Part), cudaMemcpyDeviceToDevice, st));
	MTZ_NCCL(h, ncclAllGather(h->d_xagg, h->d_xall, sizeof(Part) / 8, ncclUint64, h->xcomm, st));
	if (hop && h->xrank != 0)
		MTZ_NCCL(h, ncclRecv(h->d_carry_out, 4, ncclUint64, from, h->xcomm, st));
	int32_t rc2 = dev_finish_impl(h, nullptr, h->d_xall, (uint32_t)h->xrank, nullptr, out_bytes, carry, carry_out, true);
	if (rc2 == MTZ_OK && round_base_out != nullptr) memcpy(round_base_out, &h->h_carry[3], 32);
	return rc2;
}

static int32_t dev_finish_impl(mtz_handle *h, const uint64_t carry_in[4], const void *d_all_aggs,
    uint32_t rank, const uint64_t carry_out_in[4], size_t *out_bytes, uint64_t carry[4],
    uint64_t carry_out[4], bool xchg)
{
	CHECK_H(h);
	MTZ_CU(h, cudaSetDevice(h->device));
	cudaStream_t st = h->dv_st ? h->dv_st : h->st;
	if (d_all_aggs != nullptr) {
		if (xchg) {
			k_fold_carry<<<1, 1, 0, st>>>((const Part *)d_all_aggs, rank, h->d_carry_in, &h->d_xbase[0],
			    (uint32_t)h->xworld, &h->d_xbase[1]);
			MTZ_CU(h, cudaMemcpyAsync(&h->h_carry[3], &h->d_xbase[1], 32, cudaMemcpyDeviceToHost, st));
		} else {
			k_fold_carry<<<1, 1, 0, st>>>((const Part *)d_all_aggs, rank, h->d_carry_in);
		}
		MTZ_CU(h, cudaGetLastError());
		count_launch(h, 1);
	}
	if (carry_in != nullptr) {
		memcpy(&h->h_carry[0], carry_in, 32);
		MTZ_CU(h, cudaMemcpyAsync(h->d_carry_in, &h->h_carry[0], 32, cudaMemcpyHostToDevice, st));
	}
	if (carry_out_in != nullptr) {
		memcpy(&h->h_carry[1], carry_out_in, 32);
		MTZ_CU(h, cudaMemcpyAsync(h->d_carry_out, &h->h_carry[1], 32, cudaMemcpyHostToDevice, st));
	}
	int32_t rc = launch_scan(h, st, h->dv_sums, h->dv_nrec, h->dv_tiles, h->dv_res, 1);
	if (rc != MTZ_OK) return rc;
	MTZ_CU(h, cudaMemcpyAsync(h->dv_hres, h->dv_res, sizeof(ScanResult), cudaMemcpyDeviceToHost, st));
	MTZ_CU(h, cudaMemcpyAsync(h->d_carry_in, &h->dv_res->carry, 32, cudaMemcpyDeviceToDevice, st));
	const bool codec = is_codec_mode(h->cfg.mode) && h->dv_cb.cr != nullptr;
	const bool hop = xchg && is_codec_mode(h->cfg.mode) && (h->cfg.flags & MTZ_FLAG_DEFER_VERIFY);
	// (the 32 bytes of output checksum from the chunk before were received by the caller; after the
	// stamp chain they travel on)
	if (codec && (h->cfg.flags & MTZ_FLAG_DEFER_VERIFY) && h->dv_nrec > 0) {
		// shard mode: the stamp chain of the whole shard, from the checksum the previous
		// shard's output ended with (carry_out_in, uploaded above)
		const unsigned gp = ((unsigned)h->dv_nrec + 127u) / 128u;
		k_stamp_prep<<<gp, 128, 0, st>>>(h->dv_all_orecs, h->dv_all_osums,
		    (uint32_t)h->dv_nrec, h->dv_all_steps);
		k_stamp_chain<<<1, STAMP_THREADS, 0, st>>>(h->dv_out, h->dv_all_orecs, h->dv_all_osums,
		    h->dv_all_steps, (uint32_t)h->dv_nrec, h->d_carry_out, h->dv_cb.d_ores);
		MTZ_CU(h, cudaGetLastError());
		count_launch(h, 2);
	}
	if (hop && !(h->xflags & MTZ_XCHG_LAST))
		MTZ_NCCL(h, ncclSend(h->d_carry_out, 4, ncclUint64, (h->xrank + 1) % h->xworld, h->xcomm, st));
	if (codec) {
		MTZ_CU(h, cudaMemcpyAsync(h->dv_cb.h_cres, h->dv_cb.d_cres, sizeof(CodecResult), cudaMemcpyDeviceToHost, st));
		MTZ_CU(h, cudaMemcpyAsync(h->dv_cb.h_ores, h->dv_cb.d_ores, sizeof(ScanResult), cudaMemcpyDeviceToHost, st));
	}
	if (h->dv_bres_live)
		MTZ_CU(h, cudaMemcpyAsync(h->dv_hbres, h->dv_bres, sizeof(BlockResult), cudaMemcpyDeviceToHost, st));
	MTZ_CU(h, cudaStreamSynchronize(st));
	if (h->dv_bres_live) {
		// the block verdicts of mtz_dev_submit's records (deferred ring batches were merged at harvest)
		h->dv_bres_live = false;
		const BlockResult br = *h->dv_hbres;
		mtz_rec fr;
		fr.off = 0;
		if (br.first_bad != ~0ull)
			MTZ_CU(h, cudaMemcpy(&fr, h->dv_recs + (br.first_bad - h->dv_first), sizeof fr, cudaMemcpyDeviceToHost));
		rc = block_take(h, h->bpend, br, h->dv_in, fr.off);
		if (rc != MTZ_OK) return rc;
	}
	if (codec && h->dv_nrec > 0) {
		float cm = 0;
		if (cudaEventElapsedTime(&cm, h->dv_c0, h->dv_c1) == cudaSuccess) {
			std::lock_guard<std::mutex> g(h->stats_mu);
			h->stats.codec_ms += cm;
		}
		for (size_t i = 0; i < h->dv_k3n; i++) {
			float km = 0;
			if (cudaEventElapsedTime(&km, h->dv_k3ev[2 * i], h->dv_k3ev[2 * i + 1]) == cudaSuccess) {
				std::lock_guard<std::mutex> g(h->stats_mu);
				h->stats.k3_ms += km; h->stats.k3_launches += 1;
			}
		}
		h->dv_k3n = 0;
	}
	if (h->dv_timed) {
		float ms = 0;
		if (cudaEventElapsedTime(&ms, h->dv_k1a, h->dv_k1b) == cudaSuccess) {
			std::lock_guard<std::mutex> g(h->stats_mu);
			h->stats.k1_ms += ms; h->stats.k1_launches += 1;
		}
		h->dv_timed = false;
	}
	const ScanResult &r = *h->dv_hres;
	size_t ob = h->dv_in_bytes;
	if (carry) memcpy(carry, &r.carry, 32);
	if (carry_out) memcpy(carry_out, &r.carry, 32);
	if (codec && h->dv_nrec > 0) {
		const CodecResult &c = *h->dv_cb.h_cres;
		ob = (size_t)c.out_bytes;
		if (carry_out) memcpy(carry_out, &h->dv_cb.h_ores->carry, 32);
		if (c.bad != 0xffffffffu) {
			const uint64_t bad = h->dv_first + c.bad;
			{
				std::lock_guard<std::mutex> g(h->stats_mu);
				if (bad < h->stats.bad_record) h->stats.bad_record = bad;
			}
			return fail(h, MTZ_ECODEC, "record %llu: its frame does not decode to drr_logical_size, or no decoder "
			    "takes its compression",
			    (unsigned long long)bad);
		}
		std::lock_guard<std::mutex> g(h->stats_mu);
		h->stats.lz4_decoded += c.n_dec;
		h->stats.lz4_encoded += c.n_enc;
		h->stats.lz4_certified += c.n_cert;
		h->cstats.lz4_passed += c.n_pass;
		h->cstats.lzjb_decoded += c.n_lzjb;
		h->cstats.zle_decoded += c.n_zle;
		h->cstats.gzip_decoded += c.n_gzip;
		h->cstats.gzip_passed += c.n_gzpass;
		h->cstats.gzip_encoded += c.n_gz_enc;
	}
	if (out_bytes) *out_bytes = ob;
	rc = account_result(h, r, h->dv_first, h->dv_nrec, h->dv_in_bytes, ob, block_on(h) ? &h->bpend : nullptr);
	if (rc == MTZ_OK) h->records_done = h->dv_first + h->dv_nrec;
	if (rc == MTZ_OK && codec && h->dv_nrec > 0 && h->dv_cb.h_ores->end_seen) {
		std::lock_guard<std::mutex> g(h->stats_mu);
		h->stats.end_seen = 1;
		memcpy(h->end_ck, &h->dv_cb.h_ores->end_ck, 32);
	}
	return rc;
}

// ----------------------------------------------------- batch submission ---
static int32_t ensure_slots(mtz_handle *h)
{
	if (!h->slots.empty()) return MTZ_OK;
	const size_t cap = (size_t)h->cfg.batch_bytes + MAX_RECORD_BYTES;
	const size_t rec_cap = std::max<size_t>(4096, cap / 1024);
	// n_slots batches in flight per device; consecutive batches land on consecutive devices
	const size_t G = h->devs.size();
	h->slots.resize((size_t)h->cfg.n_slots * G);
	for (size_t k = 0; k < h->slots.size(); k++) {
		Slot &s = h->slots[k];
		int32_t rc = alloc_slot(h, s, (int)(k % G), cap, rec_cap);
		if (rc != MTZ_OK) return rc;
		if (is_codec_mode(h->cfg.mode)) {
			s.out_cap = cap;
			MTZ_CU(h, cudaMalloc(&s.d_out, cap + 512));
		}
		if (is_codec_mode(h->cfg.mode) || block_frames_on(h)) {
			rc = codec_alloc(h, s.cb, rec_cap, cap + rec_cap * 48);
			if (rc != MTZ_OK) return rc;
		}
	}
	MTZ_CU(h, cudaSetDevice(h->device));
	return MTZ_OK;
}

// Batch assembly shared by the bulk and the streaming paths: decides whether the
// record whose header is `hdr` still fits the batch being cut for slot s.
struct BatchCut {
	size_t cnt = 0, in_bytes = 0, budget = 0; uint64_t writes = 0;
	bool emit_pre = false;           // COMPRESS: the batch starts with BEGIN, its output gets a preamble
	uint32_t pre_flags = 0;
};

// state of the lz4-stage-v1 wire framing on the INPUT side (DECOMPRESS): a preamble was read and
// the BEGIN it announces has not arrived yet
struct WireState { bool pre_seen = false; uint32_t pre_flags = 0; };

static void wire_preamble(uint8_t out[WIRE_PRE_BYTES], uint32_t flags)
{
	memset(out, 0, WIRE_PRE_BYTES);
	const uint64_t m = WIRE_MAGIC;
	const uint32_t v = WIRE_VERSION;
	memcpy(out, &m, 8); memcpy(out + 8, &v, 4); memcpy(out + 12, &flags, 4);
}

// 1: a preamble this side speaks (flags out); 0: not a preamble; <0: a preamble of a version or
// with capability bits this side does not know.  WIRE_F_GZIP is known only to a DECOMPRESS opened with
// MTZ_FLAG_GZIP_WIRE: any other receiver refuses the wire rather than hand gzip records on.
static int wire_parse(const mtz_handle *h, const uint8_t *p, uint32_t *flags)
{
	const uint32_t known = WIRE_F_ORIG_LZ4 | (gzwire_on(h) ? WIRE_F_GZIP : 0u);
	if (rd64(p) != WIRE_MAGIC) return 0;
	if (rd32(p + 8) != WIRE_VERSION || (rd32(p + 12) & ~known) != 0) return -1;
	for (unsigned k = 16; k < WIRE_PRE_BYTES; k++) if (p[k] != 0) return -1;
	*flags = rd32(p + 12);
	return 1;
}

// The preamble's WIRE_F_ORIG_LZ4: the stream `zfs send` without -c would have produced carries the
// LZ4 feature.  -c alone sets it whenever the pool's lz4 feature is active, without -c only -e
// (EMBED_DATA) does ([EXTERNAL] dmu_send.c), so a compressed stream keeps it only with EMBED_DATA.
static uint32_t wire_orig_lz4(uint64_t feat)
{
	return (feat & FEAT_LZ4) && (!(feat & FEAT_COMPRESSED) || (feat & FEAT_EMBED_DATA)) ? WIRE_F_ORIG_LZ4 : 0u;
}

// returns 1 accepted, 0 batch is full (cut first), <0 error (already reported)
static int32_t batch_accept(mtz_handle *h, const Slot &s, BatchCut &bc, const uint8_t *hdr,
    int64_t pl, uint32_t ls, uint32_t comp, uint64_t stream_off, mtz_rec *out, WireState *ws)
{
	const size_t rl = DRR_HDR + (size_t)pl;
	const bool codec = is_codec_mode(h->cfg.mode);
	const uint32_t type = rd32(hdr);
	size_t cost = rl;
	if (codec) cost = DRR_HDR + std::max<size_t>((size_t)pl, ls) + 48;
	if (cost > s.cap)
		return fail(h, MTZ_ENOSPC, "record of %zu bytes at stream offset %llu exceeds the batch slot",
		    cost, (unsigned long long)stream_off);
	if (bc.cnt > 0 && (bc.budget + cost > s.cap || bc.cnt >= s.rec_cap)) return 0;
	uint64_t resv = 0;
	if (ws->pre_seen && type != 0)
		return fail(h, MTZ_EFORMAT, "wire preamble at stream offset %llu is not followed by DRR_BEGIN",
		    (unsigned long long)stream_off);
	if (codec && type == 0) {
		// BEGIN: the modes are only defined on the streams oracle/stream.c accepts
		const uint64_t vi = rd64(hdr + 16);
		const uint64_t feat = (vi >> 2) & ((1ull << 30) - 1ull);
		if (h->cfg.mode == MTZ_MODE_COMPRESS) {
			if ((feat & FEAT_COMPRESSED) && !cin_on(h))
				return fail(h, MTZ_EINVAL, "COMPRESS: stream is already compressed");
			// the lz4-stage-v1 wire puts a preamble in front of every BEGIN: BEGIN opens its batch
			if (bc.cnt > 0) return 0;
			bc.emit_pre = true;
			bc.pre_flags = wire_orig_lz4(feat) | (gzwire_on(h) || gzenc_on(h) ? WIRE_F_GZIP : 0u);
		} else if (h->cfg.mode == MTZ_MODE_DECOMPRESS) {
			if (!ws->pre_seen)
				return fail(h, MTZ_EINVAL, "DECOMPRESS: stream was not produced by the COMPRESS stage");
			resv = ws->pre_flags;
			ws->pre_seen = false;
		}
	}
	mtz_rec r;
	r.off = bc.in_bytes; r.payload = (uint32_t)pl; r.type = type;
	r.lsize = ls; r.comp = comp; r.resv = resv;
	*out = r;
	bc.cnt++; bc.in_bytes += rl; bc.budget += cost;
	if (type == 3) bc.writes++;
	return 1;
}

// Wait for a slot's kernels, fold its verdict into the handle.
static int32_t harvest(mtz_handle *h, Slot &s)
{
	if (!s.busy) return MTZ_OK;
	MTZ_CU(h, cudaEventSynchronize(s.ev_done));
	s.busy = false;
	float ms = 0, k1 = 0, cm = 0, k3 = 0;
	const bool k3ok = s.k3_timed && cudaEventElapsedTime(&k3, s.ev_k3a, s.ev_k3b) == cudaSuccess;
	s.k3_timed = false;
	cudaEventElapsedTime(&ms, s.ev_start, s.ev_done);
	const bool codec = is_codec_mode(h->cfg.mode);
	const bool k1ok = s.nrec > 0 && cudaEventElapsedTime(&k1, s.ev_k1a, s.ev_k1b) == cudaSuccess;
	const bool cok = codec && s.nrec > 0 && cudaEventElapsedTime(&cm, s.ev_c0, s.ev_c1) == cudaSuccess;
	{
		std::lock_guard<std::mutex> g(h->stats_mu);
		h->stats.gpu_ms += ms;
		h->stats.write_records += s.writes;
		if (k1ok) { h->stats.k1_ms += k1; h->stats.k1_launches += 1; }
		if (cok) h->stats.codec_ms += cm;
		if (k3ok) { h->stats.k3_ms += k3; h->stats.k3_launches += 1; }
	}
	BlockPending bp;
	if (block_on(h) && s.nrec > 0) {
		const BlockResult &br = *s.h_bres;
		const uint64_t off = br.first_bad != ~0ull ? s.h_recs[br.first_bad - s.first_rec].off : 0;
		// deferred batches: the verdict waits for mtz_dev_finish, with the stream verdict
		int32_t rc = block_take(h, (h->cfg.flags & MTZ_FLAG_DEFER_VERIFY) ? h->bpend : bp, br, s.d_in, off);
		if (rc != MTZ_OK) return rc;
	}
	if (h->cfg.mode == MTZ_MODE_PASSTHROUGH || (h->cfg.flags & MTZ_FLAG_DEFER_VERIFY)) {
		std::lock_guard<std::mutex> g(h->stats_mu);
		h->stats.batches += 1; h->stats.bytes_in += s.bytes; h->stats.bytes_out += s.out_bytes;
		h->stats.records += s.nrec;
		return MTZ_OK;
	}
	if (codec && s.nrec > 0) {
		const CodecResult &c = *s.cb.h_cres;
		s.out_bytes = (size_t)c.out_bytes;
		if (c.bad != 0xffffffffu) {
			const uint64_t bad = s.first_rec + c.bad;
			{
				std::lock_guard<std::mutex> g(h->stats_mu);
				if (bad < h->stats.bad_record) h->stats.bad_record = bad;
			}
			return fail(h, MTZ_ECODEC, "record %llu: its frame does not decode to drr_logical_size, or no decoder "
			    "takes its compression",
			    (unsigned long long)bad);
		}
		std::lock_guard<std::mutex> g(h->stats_mu);
		h->stats.lz4_decoded += c.n_dec;
		h->stats.lz4_encoded += c.n_enc;
		h->stats.lz4_certified += c.n_cert;
		h->cstats.lz4_passed += c.n_pass;
		h->cstats.lzjb_decoded += c.n_lzjb;
		h->cstats.zle_decoded += c.n_zle;
		h->cstats.gzip_decoded += c.n_gzip;
		h->cstats.gzip_passed += c.n_gzpass;
		h->cstats.gzip_encoded += c.n_gz_enc;
	}
	int32_t rc = account_result(h, *s.h_res, s.first_rec, s.nrec, s.bytes, s.out_bytes,
	    block_on(h) ? &bp : nullptr);
	if (rc == MTZ_OK && codec && s.nrec > 0 && s.cb.h_ores->end_seen) {
		std::lock_guard<std::mutex> g(h->stats_mu);
		h->stats.end_seen = 1;
		memcpy(h->end_ck, &s.cb.h_ores->end_ck, 32);     // END checksum of the OUTPUT stream
	}
	return rc;
}

// The block check of slot s's batch as far as its input goes, `isums` = the input's sums: the
// results reset, then VERIFY's frames and their check (launch_block_frames) or the check of the input
// records.  The codec modes check their records after the output's sums (codec_launch_post).
static int32_t launch_block_input(mtz_handle *h, Slot &s, const RecSums *isums)
{
	if (!block_on(h) || s.nrec == 0) return MTZ_OK;
	int32_t rc = block_reset(h, s.st, s.d_bres);
	if (rc == MTZ_OK && block_frames_on(h))
		rc = launch_block_frames(h, s.st, s.cb, s.d_in, s.d_recs, isums, s.nrec, 0,
		    all_compact_blocks(s.h_recs, s.nrec), s.first_rec, s.d_bres);
	else if (rc == MTZ_OK && !is_codec_mode(h->cfg.mode))
		rc = launch_block(h, s.st, s.d_in, s.d_recs, isums, nullptr, nullptr, nullptr, s.nrec, s.first_rec, s.d_bres);
	return rc;
}

// Enqueue one batch: the bytes come from up to two host pieces (ring wrap),
// s.h_recs[0..nrec) is already filled with batch-relative offsets.
static int32_t submit_batch(mtz_handle *h, Slot &s, const uint8_t *p0, size_t n0,
    const uint8_t *p1, size_t n1, size_t nrec, uint64_t abs_off, uint8_t *host_out)
{
	const size_t bytes = n0 + n1;
	DevCtx &dc = h->devs[s.di];
	s.nrec = nrec; s.bytes = bytes; s.out_bytes = bytes; s.in_off = abs_off;
	s.first_rec = h->records_done;
	h->records_done += nrec;
	MTZ_CU(h, cudaSetDevice(dc.device));
	MTZ_CU(h, cudaEventRecord(s.ev_start, s.st));
	if (nrec > 0)
		MTZ_CU(h, cudaMemcpyAsync(s.d_recs, s.h_recs, nrec * sizeof(mtz_rec), cudaMemcpyHostToDevice, s.st));
	if (n0) MTZ_CU(h, cudaMemcpyAsync(s.d_in, p0, n0, cudaMemcpyHostToDevice, s.st));
	if (n1) MTZ_CU(h, cudaMemcpyAsync(s.d_in + n0, p1, n1, cudaMemcpyHostToDevice, s.st));
	MTZ_CU(h, cudaEventRecord(s.ev_h2d, s.st));
	int32_t rc = MTZ_OK;
	if (h->cfg.mode == MTZ_MODE_VERIFY && (h->cfg.flags & MTZ_FLAG_DEFER_VERIFY)) {
		// shard mode: sums accumulate in the handle-wide table; verdict later
		rc = ensure_dv_sums(h, h->dv_nrec + nrec, s.st);
		if (rc != MTZ_OK) return rc;
		rc = launch_k1(h, s.st, s.d_in, s.d_recs, nrec, h->dv_sums + h->dv_nrec, s.ev_k1a, s.ev_k1b,
		    nrec ? bytes / nrec : 0);
		if (rc != MTZ_OK) return rc;
		// the block check needs no running checksum: it runs now, its verdict waits with the stream's
		rc = launch_block_input(h, s, h->dv_sums + h->dv_nrec);
		if (rc != MTZ_OK) return rc;
		if (h->dv_nrec == 0) h->dv_first = s.first_rec;
		h->dv_nrec += nrec; h->dv_in_bytes += bytes; h->dv_st = h->st;
	} else if (h->cfg.mode != MTZ_MODE_PASSTHROUGH) {
		// every mode verifies the INPUT stream's checksums
		rc = launch_k1(h, s.st, s.d_in, s.d_recs, nrec, s.d_sums, s.ev_k1a, s.ev_k1b,
		    nrec ? bytes / nrec : 0);
		if (rc != MTZ_OK) return rc;
		rc = launch_block_input(h, s, s.d_sums);
		if (rc != MTZ_OK) return rc;
		if (is_codec_mode(h->cfg.mode)) {
			rc = codec_reset(h, s.st, s.cb);
			if (rc != MTZ_OK) return rc;
			// K2/K3 of this batch overlap the previous batch's checksum chains
			const bool enc = h->cfg.mode != MTZ_MODE_DECOMPRESS && nrec > 0;
			rc = codec_launch_pre(h, s.st, s.cb, s.d_in, s.d_recs, nrec, s.ev_c0, s.ev_c1,
			    all_compact_blocks(s.h_recs, nrec), enc ? s.ev_k3a : nullptr, enc ? s.ev_k3b : nullptr, s.st_k3);
			if (rc != MTZ_OK) return rc;
			s.k3_timed = enc;
		}
		// the running checksums arrive with the previous batch: wait for its chain and, when it
		// ran on another GPU of the group, fetch the 64 bytes over NVLink / PCIe
		if (h->prev_scan_slot >= 0) {
			const Slot &ps = h->slots[(size_t)h->prev_scan_slot];
			MTZ_CU(h, cudaStreamWaitEvent(s.st, ps.ev_scan, 0));
			if (ps.di != s.di) {
				const DevCtx &pd = h->devs[ps.di];
				MTZ_CU(h, cudaMemcpyPeerAsync(dc.d_carry_in, dc.device, pd.d_carry_in, pd.device, sizeof(Ck4), s.st));
				MTZ_CU(h, cudaMemcpyPeerAsync(dc.d_carry_out, dc.device, pd.d_carry_out, pd.device, sizeof(Ck4), s.st));
			}
		}
		rc = launch_scan(h, s.st, s.d_sums, nrec, s.d_tiles, s.d_res, 1, dc.d_carry_in);
		if (rc != MTZ_OK) return rc;
		MTZ_CU(h, cudaMemcpyAsync(dc.d_carry_in, &s.d_res->carry, 32, cudaMemcpyDeviceToDevice, s.st));
		if (is_codec_mode(h->cfg.mode)) {
			rc = codec_launch_post(h, s.st, s.cb, s.d_in, s.d_recs, nrec, s.d_out, 0u, nullptr, nullptr,
			    dc.d_carry_out, s.d_sums, s.first_rec, (block_on(h) && nrec > 0) ? s.d_bres : nullptr);
			if (rc != MTZ_OK) return rc;
			MTZ_CU(h, cudaMemcpyAsync(s.cb.h_cres, s.cb.d_cres, sizeof(CodecResult), cudaMemcpyDeviceToHost, s.st));
			MTZ_CU(h, cudaMemcpyAsync(s.cb.h_ores, s.cb.d_ores, sizeof(ScanResult), cudaMemcpyDeviceToHost, s.st));
		}
		MTZ_CU(h, cudaEventRecord(s.ev_scan, s.st));
		h->prev_scan_slot = (int)(&s - h->slots.data());
		MTZ_CU(h, cudaMemcpyAsync(s.h_res, s.d_res, sizeof(ScanResult), cudaMemcpyDeviceToHost, s.st));
	}
	if (block_on(h) && nrec > 0)
		MTZ_CU(h, cudaMemcpyAsync(s.h_bres, s.d_bres, sizeof(BlockResult), cudaMemcpyDeviceToHost, s.st));
	if (host_out != nullptr && !is_codec_mode(h->cfg.mode))
		MTZ_CU(h, cudaMemcpyAsync(host_out, s.d_in, bytes, cudaMemcpyDeviceToHost, s.st));
	MTZ_CU(h, cudaEventRecord(s.ev_done, s.st));
	s.busy = true;
	return MTZ_OK;
}

// -------------------------------------------------------- bulk host API ---
int32_t mtz_process_host(mtz_handle *h, const void *in, size_t n, void *out, size_t out_cap,
    size_t *out_n)
{
	CHECK_H(h);
	if (in == nullptr && n != 0) return MTZ_EINVAL;
	const bool codec = is_codec_mode(h->cfg.mode);
	if (codec && (h->cfg.flags & MTZ_FLAG_DEFER_VERIFY))
		return fail(h, MTZ_EINVAL, "deferred verification is a VERIFY-mode feature");
	if (!codec && out != nullptr && out != in && out_cap < n)
		return fail(h, MTZ_ENOSPC, "output buffer smaller than the stream");
	if (codec && out == nullptr)
		return fail(h, MTZ_EINVAL, "codec modes need an output buffer");
	MTZ_CU(h, cudaSetDevice(h->device));
	int32_t rc = ensure_slots(h);
	if (rc != MTZ_OK) return rc;

	const uint8_t *src = (const uint8_t *)in;
	const bool parse = h->cfg.mode != MTZ_MODE_PASSTHROUGH;
	size_t off = 0, out_pos = 0;
	uint64_t b = 0;
	// retire the batch that occupies slot s: verdict, then (codec) its output bytes
	auto retire = [&](Slot &s) -> int32_t {
		const bool was_busy = s.busy;
		int32_t r = harvest(h, s);
		if (r != MTZ_OK || !was_busy || !codec) return r;
		const size_t pre = s.emit_pre ? WIRE_PRE_BYTES : 0;
		if (out_pos + pre + s.out_bytes > out_cap)
			return fail(h, MTZ_ENOSPC, "output buffer too small (%zu needed so far)", out_pos + pre + s.out_bytes);
		if (pre) {
			wire_preamble((uint8_t *)out + out_pos, s.pre_flags);
			out_pos += pre;
			std::lock_guard<std::mutex> g(h->stats_mu);
			h->stats.bytes_out += pre;
		}
		MTZ_CU(h, cudaSetDevice(h->devs[s.di].device));
		// issued, not awaited: the copy-out of batch b overlaps the parse + submit of the batches
		// behind it; the slot is only reused (or the call returns) after `drain_d2h`
		MTZ_CU(h, cudaMemcpyAsync((uint8_t *)out + out_pos, s.d_out, s.out_bytes, cudaMemcpyDeviceToHost, s.st));
		MTZ_CU(h, cudaEventRecord(s.ev_done, s.st));
		s.d2h_pending = true;
		out_pos += s.out_bytes;
		return MTZ_OK;
	};
	auto drain_d2h = [&](Slot &s) -> int32_t {
		if (!s.d2h_pending) return MTZ_OK;
		s.d2h_pending = false;
		MTZ_CU(h, cudaEventSynchronize(s.ev_done));
		return MTZ_OK;
	};
	// Output order == submission order.  Batches are retired (verdict folded in, output copy ISSUED)
	// in order as soon as they are done -- looked at every iteration, not only when their slot
	// comes round again: on a device group several GPUs' output copies then overlap on their own
	// PCIe links instead of queueing behind one host wait per batch.  A slot is reused once its
	// batch is retired and its copy has landed.
	const size_t NS = h->slots.size();
	uint64_t nr = 0;                                  // batches retired so far
	auto retire_next = [&](bool block) -> int32_t {   // 1 = the oldest batch is still running
		Slot &rs = h->slots[nr % NS];
		if (!block && rs.busy && cudaEventQuery(rs.ev_done) == cudaErrorNotReady) return 1;
		int32_t r = retire(rs);
		if (r == MTZ_OK) nr++;
		return r;
	};
	WireState ws;
	while (off < n && rc == MTZ_OK) {
		Slot &s = h->slots[b % NS];
		while (rc == MTZ_OK && nr < b) {
			const int32_t r = retire_next(false);
			if (r == 1) break;
			rc = r;
		}
		while (rc == MTZ_OK && nr + NS <= b) rc = retire_next(true);
		if (rc == MTZ_OK) rc = drain_d2h(s);
		if (rc != MTZ_OK) break;
		BatchCut bc;
		if (!parse) {
			bc.in_bytes = std::min(n - off, std::min((size_t)h->cfg.batch_bytes, s.cap));
		} else {
			while (off + bc.in_bytes < n) {
				const size_t at = off + bc.in_bytes;
				const uint8_t *hp = src + at;
				uint32_t ls, comp;
				if (h->cfg.mode == MTZ_MODE_DECOMPRESS && !ws.pre_seen && n - at >= WIRE_PRE_BYTES &&
				    rd64(hp) == WIRE_MAGIC) {
					// the preamble of the lz4-stage-v1 wire: stripped here, between two batches
					if (bc.cnt > 0) break;
					if (wire_parse(h, hp, &ws.pre_flags) < 0) {
						rc = fail(h, MTZ_EFORMAT, "unsupported wire version / capability in the preamble at offset %zu", at);
						break;
					}
					ws.pre_seen = true;
					off += WIRE_PRE_BYTES;
					{
						std::lock_guard<std::mutex> g(h->stats_mu);
						h->stats.bytes_in += WIRE_PRE_BYTES;
					}
					continue;
				}
				if (n - at < DRR_HDR) { rc = fail(h, MTZ_EFORMAT, "truncated record header at offset %zu", at); break; }
				const int64_t pl = drr_payload(hp, &ls, &comp);
				if (pl < 0) { rc = fail(h, MTZ_EFORMAT, "malformed record header at offset %zu", at); break; }
				if ((uint64_t)pl > n - at - DRR_HDR) { rc = fail(h, MTZ_EFORMAT, "truncated payload at offset %zu", at); break; }
				const int32_t a = batch_accept(h, s, bc, hp, pl, ls, comp, at, &s.h_recs[bc.cnt], &ws);
				if (a < 0) { rc = a; break; }
				if (a == 0) break;
				if (bc.budget >= (size_t)h->cfg.batch_bytes) break;
			}
		}
		if (rc != MTZ_OK) break;
		if (bc.cnt == 0 && bc.in_bytes == 0 && parse) continue;      // (only a preamble was consumed)
		s.writes = bc.writes;
		s.emit_pre = bc.emit_pre; s.pre_flags = bc.pre_flags;
		uint8_t *ho = (!codec && out != nullptr && out != in) ? (uint8_t *)out + off : nullptr;
		rc = submit_batch(h, s, src + off, bc.in_bytes, nullptr, 0, bc.cnt, off, ho);
		off += bc.in_bytes;
		b++;
	}
	// drain in submission order
	while (nr < b) {
		int32_t r2 = retire_next(true);
		if (r2 != MTZ_OK) { if (rc == MTZ_OK) rc = r2; nr++; }
	}
	for (size_t k = 0; k < NS; k++) {
		int32_t r2 = drain_d2h(h->slots[k]);
		if (rc == MTZ_OK) rc = r2;
	}
	cudaSetDevice(h->device);
	if (out_n) *out_n = (rc != MTZ_OK) ? 0 : (codec ? out_pos : n);
	return rc;
}

} // extern "C"

// ======================================================= streaming engine ==
#include "mtz_engine.inl"
extern "C" {

// ---------------------------------------------------- LZ4 kernel entries ---
// One warp per record, one CTA per LZ4_WARPS records: CTAs that live for one record each free
// their SM slot every few microseconds somewhere on the chip, so kernels of other streams
// interleave with a long encode and the hardware balances ragged records (+1-2 % over the
// one-wave grid-stride launch, which MTZ_LZ4_PERSISTENT=1 restores for experiments).
static bool lz4_persistent()
{
	static const bool p = [] { const char *e = getenv("MTZ_LZ4_PERSISTENT"); return e != nullptr && atoi(e) != 0; }();
	return p;
}
static int32_t lz4_grid(mtz_handle *h, uint32_t njobs, int warps_per_sm)
{
	const uint32_t blocks_needed = (njobs + LZ4_WARPS - 1) / LZ4_WARPS;
	if (warps_per_sm <= 0) return (int32_t)std::max(1u, blocks_needed);
	const uint32_t cap = (uint32_t)h->sm_count * (uint32_t)(warps_per_sm / LZ4_WARPS);
	return (int32_t)std::max(1u, std::min(blocks_needed, cap));
}

// K2 on `st`, which belongs to the CURRENT device (the caller selected it: a slot of the device
// group, or devs[0] for the exported entry)
static int32_t launch_k2(mtz_handle *h, cudaStream_t st, const void *d_src, void *d_dst, mtz_job *d_jobs,
    uint32_t njobs, const mtz_job *seq_jobs, uint32_t *seq_n)
{
	if (njobs == 0) return MTZ_OK;
	k2_lz4_decode<<<lz4_grid(h, njobs, lz4_persistent() ? 64 : 0), LZ4_THREADS, 0, st>>>((const uint8_t *)d_src,
	    (uint8_t *)d_dst, d_jobs, njobs, seq_jobs, seq_n);
	MTZ_CU(h, cudaGetLastError());
	count_launch(h, 1);
	return MTZ_OK;
}

int32_t mtz_k_lz4_decode(mtz_handle *h, const void *d_src, void *d_dst, mtz_job *d_jobs,
    uint32_t njobs, void *cuda_stream)
{
	CHECK_H(h);
	if (njobs == 0) return MTZ_OK;
	MTZ_CU(h, cudaSetDevice(h->device));
	cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : h->st;
	return launch_k2(h, st, d_src, d_dst, d_jobs, njobs, nullptr, nullptr);
}

// Function attributes are per DEVICE (and per context): set them for the current device of
// every handle at open time, not once per process -- a second GPU opened in the same process
// would otherwise launch k3_lz4_encode<false> with 64 KiB of dynamic shared memory it never
// opted into.  Idempotent, so concurrent handles on one device do not need a lock.
static int32_t k3_set_attributes(mtz_handle *h)
{
	MTZ_CU(h, cudaFuncSetAttribute(k3_lz4_encode<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
	    (int)((size_t)K3_WARPS * LZ4_TAB_COMPACT_WORDS * 4)));
	MTZ_CU(h, cudaFuncSetAttribute(k3_lz4_encode<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
	    (int)((size_t)K3_WARPS * LZ4_TAB_BIG_WORDS * 4)));
	MTZ_CU(h, cudaFuncSetAttribute(k3c_lz4_certify<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
	    (int)((size_t)K3_WARPS * LZ4_TAB_COMPACT_WORDS * 4)));
	MTZ_CU(h, cudaFuncSetAttribute(k3c_lz4_certify<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
	    (int)((size_t)K3_WARPS * LZ4_TAB_BIG_WORDS * 4)));
	{
		// experiments: a smaller carve-out trades certificate warps per SM for L1
		const char *c = getenv("MTZ_K3C_CARVEOUT");
		if (c != nullptr && atoi(c) > 0) {
			MTZ_CU(h, cudaFuncSetAttribute(k3c_lz4_certify<true>, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(c)));
			MTZ_CU(h, cudaFuncSetAttribute(k3c_lz4_certify<false>, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(c)));
		}
	}
	// all of the unified L1/shared array as shared memory: K3 is bound by records in
	// flight (24 tables of 8.5 KiB per SM, which a 75 % carve-out cannot hold).
	// MTZ_K3_CARVEOUT overrides for experiments.
	const char *e = getenv("MTZ_K3_CARVEOUT");
	const int pct = e ? atoi(e) : 100;
	MTZ_CU(h, cudaFuncSetAttribute(k3_lz4_encode<true>, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
	MTZ_CU(h, cudaFuncSetAttribute(k3_lz4_encode<false>, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
	return MTZ_OK;
}

// compact = every block is 64 KiB+11 .. 128 KiB: 8.5 KiB tables, more warps per SM.  `count` = the
// launch is counted in mtz_stats.kernel_launches (not the block check's, launch_block_frames)
static int32_t launch_k3(mtz_handle *h, cudaStream_t st, const void *d_src, void *d_dst,
    mtz_job *d_jobs, uint32_t njobs, bool compact, const uint32_t *skip, bool count)
{
	const size_t tabw = compact ? LZ4_TAB_COMPACT_WORDS : LZ4_TAB_BIG_WORDS;
	const size_t smem = (size_t)K3_WARPS * tabw * sizeof(uint32_t);
	int blocks_per_sm = (int)((227u * 1024u) / (smem + 1024));
	{
		// experiments only (tools/k3_bound.py): fewer encoder CTAs per SM than the tables allow
		const char *e = getenv("MTZ_K3_BLOCKS_PER_SM");
		if (e && atoi(e) > 0) blocks_per_sm = std::min(blocks_per_sm, atoi(e));
	}
	const uint32_t need = (njobs + K3_WARPS - 1) / K3_WARPS;
	const int grid = (int)std::max(1u, lz4_persistent() ? std::min(need, (uint32_t)h->sm_count * (uint32_t)blocks_per_sm) : need);
	if (compact)
		k3_lz4_encode<true><<<grid, K3_THREADS, smem, st>>>((const uint8_t *)d_src, (uint8_t *)d_dst, d_jobs, njobs, skip);
	else
		k3_lz4_encode<false><<<grid, K3_THREADS, smem, st>>>((const uint8_t *)d_src, (uint8_t *)d_dst, d_jobs, njobs, skip);
	MTZ_CU(h, cudaGetLastError());
	if (count) count_launch(h, 1);
	return MTZ_OK;
}

// K3c over the (sub-)batch: verdicts into cb.cert, which K3 (skip) and the assembler then read
static int32_t launch_k3c(mtz_handle *h, cudaStream_t st, CodecBufs &cb, uint32_t njobs, bool compact)
{
	if (njobs == 0) return MTZ_OK;
	const size_t tabw = compact ? LZ4_TAB_COMPACT_WORDS : LZ4_TAB_BIG_WORDS;
	const size_t smem = (size_t)K3_WARPS * tabw * sizeof(uint32_t);
	const int grid = (int)((njobs + K3_WARPS - 1) / K3_WARPS);
	if (compact)
		k3c_lz4_certify<true><<<grid, K3_THREADS, smem, st>>>(cb.dec, cb.enc, cb.seq_n, cb.cert, njobs);
	else
		k3c_lz4_certify<false><<<grid, K3_THREADS, smem, st>>>(cb.dec, cb.enc, cb.seq_n, cb.cert, njobs);
	MTZ_CU(h, cudaGetLastError());
	count_launch(h, 1);
	return MTZ_OK;
}

int32_t mtz_k_lz4_encode(mtz_handle *h, const void *d_src, void *d_dst, mtz_job *d_jobs,
    uint32_t njobs, void *cuda_stream)
{
	CHECK_H(h);
	if (njobs == 0) return MTZ_OK;
	MTZ_CU(h, cudaSetDevice(h->device));
	cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : h->st;
	// MTZ_K3_FORCE_COMPACT: the caller vouches that every job is a 128 KiB-class block (experiments)
	const char *e = getenv("MTZ_K3_FORCE_COMPACT");
	return launch_k3(h, st, d_src, d_dst, d_jobs, njobs, e != nullptr && atoi(e) != 0);
}

// K3, then k_deflate_from_lz4 on the same stream: K3's frames go to a scratch of the handle at the jobs'
// dst_off, the zlib frames to d_dst.  Reads the job table to size that scratch, so it synchronises.
int32_t mtz_k_gzip_encode(mtz_handle *h, const void *d_src, void *d_dst, mtz_job *d_jobs,
    uint32_t njobs, void *cuda_stream)
{
	CHECK_H(h);
	if (njobs == 0) return MTZ_OK;
	if (((uintptr_t)d_dst & 3u) != 0) return fail(h, MTZ_EINVAL, "mtz_k_gzip_encode: d_dst must be 4-byte aligned");
	MTZ_CU(h, cudaSetDevice(h->device));
	cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : h->st;
	std::vector<mtz_job> jobs(njobs);
	MTZ_CU(h, cudaMemcpyAsync(jobs.data(), d_jobs, njobs * sizeof(mtz_job), cudaMemcpyDeviceToHost, st));
	MTZ_CU(h, cudaStreamSynchronize(st));
	size_t need = 0;
	for (const mtz_job &j : jobs) {
		if (j.lsize == 0) continue;
		if ((j.dst_off & 3u) != 0) return fail(h, MTZ_EINVAL, "mtz_k_gzip_encode: every dst_off must be 4-byte aligned");
		need = std::max<size_t>(need, (size_t)j.dst_off + j.lsize);
	}
	if (need > h->k_gz_lz_cap) {
		if (h->k_gz_lz) MTZ_CU(h, cudaFree(h->k_gz_lz));
		h->k_gz_lz = nullptr; h->k_gz_lz_cap = 0;
		MTZ_CU(h, cudaMalloc(&h->k_gz_lz, need + 16));
		h->k_gz_lz_cap = need;
	}
	int32_t rc = launch_k3(h, st, d_src, h->k_gz_lz, d_jobs, njobs, false);
	if (rc != MTZ_OK) return rc;
	k_deflate_from_lz4<<<defl_grid(h, njobs), DEFL_THREADS, 0, st>>>(d_jobs, d_jobs, njobs, (uint64_t)(uintptr_t)d_src,
	    (uint64_t)(uintptr_t)h->k_gz_lz, (uint64_t)(uintptr_t)d_dst, false);
	MTZ_CU(h, cudaGetLastError());
	count_launch(h, 1);
	return MTZ_OK;
}

// K3h over njobs jobs with `tabs` (hc_tab_bytes): the persistent grid has exactly the warps the
// tables were sized for, at most
static int32_t launch_k3h(mtz_handle *h, cudaStream_t st, const void *d_src, void *d_dst,
    mtz_job *d_jobs, uint32_t njobs, uint32_t *tabs)
{
	if (njobs == 0) return MTZ_OK;
	const uint32_t need = (njobs + LZ4HC_WARPS - 1) / LZ4HC_WARPS;
	const int grid = (int)std::min(need, (uint32_t)h->sm_count * (uint32_t)LZ4HC_CTAS_PER_SM);
	k3h_lz4hc_encode<<<grid, LZ4HC_THREADS, 0, st>>>((const uint8_t *)d_src, (uint8_t *)d_dst, d_jobs, njobs, tabs);
	MTZ_CU(h, cudaGetLastError());
	count_launch(h, 1);
	return MTZ_OK;
}

int32_t mtz_k_lz4hc_encode(mtz_handle *h, const void *d_src, void *d_dst, mtz_job *d_jobs,
    uint32_t njobs, void *cuda_stream)
{
	CHECK_H(h);
	if (njobs == 0) return MTZ_OK;
	MTZ_CU(h, cudaSetDevice(h->device));
	cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : h->st;
	if (h->k_hc_tab == nullptr) MTZ_CU(h, cudaMalloc(&h->k_hc_tab, hc_tab_bytes(h)));
	return launch_k3h(h, st, d_src, d_dst, d_jobs, njobs, h->k_hc_tab);
}

// ------------------------------------------------------- GPU-side parse ---
int32_t mtz_dev_index(mtz_handle *h, const void *d_in, size_t n, mtz_rec *d_recs, size_t cap,
    size_t *nrec, size_t *consumed, void *cuda_stream)
{
	CHECK_H(h);
	if (d_in == nullptr || d_recs == nullptr) return MTZ_EINVAL;
	if (((uintptr_t)d_in & 3) != 0) return fail(h, MTZ_EINVAL, "d_in must be 4-byte aligned");
	MTZ_CU(h, cudaSetDevice(h->device));
	cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : h->st;
	if (h->d_ires == nullptr) {
		MTZ_CU(h, cudaMalloc(&h->d_ires, sizeof(IndexResult)));
		MTZ_CU(h, cudaHostAlloc(&h->h_ires, sizeof(IndexResult), cudaHostAllocDefault));
		MTZ_CU(h, cudaMalloc(&h->d_ishared, sizeof(IndexShared)));
	}
	MTZ_CU(h, cudaMemsetAsync(h->d_ishared, 0xff, sizeof(IndexShared), st));
	{
		// cooperative launch: one CTA per SM (1024 threads x 64 regs fill the register file)
		const uint8_t *a0 = (const uint8_t *)d_in;
		uint64_t a1 = (uint64_t)n, a3 = (uint64_t)cap;
		mtz_rec *a2 = d_recs;
		IndexResult *a4 = h->d_ires;
		IndexShared *a5 = h->d_ishared;
		void *args[] = { &a0, &a1, &a2, &a3, &a4, &a5 };
		MTZ_CU(h, cudaLaunchCooperativeKernel((void *)k_index, dim3((unsigned)h->sm_count),
		    dim3(INDEX_THREADS), args, 0, st));
	}
	count_launch(h, 1);
	MTZ_CU(h, cudaMemcpyAsync(h->h_ires, h->d_ires, sizeof(IndexResult), cudaMemcpyDeviceToHost, st));
	MTZ_CU(h, cudaStreamSynchronize(st));
	if (nrec) *nrec = (size_t)h->h_ires->nrec;
	if (consumed) *consumed = (size_t)h->h_ires->consumed;
	if (h->h_ires->status == MTZ_EFORMAT)
		return fail(h, MTZ_EFORMAT, "malformed record header at stream offset %llu",
		    (unsigned long long)h->h_ires->consumed);
	if (h->h_ires->status == MTZ_ENOSPC) return MTZ_ENOSPC;     // not sticky: caller may retry bigger
	return MTZ_OK;
}

} // extern "C"
