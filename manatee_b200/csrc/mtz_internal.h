// mtz_internal.h -- private state of a libmanatee_gpu handle.
#pragma once
#include <atomic>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include <cuda_runtime.h>
#include "mtz_nccl.h"
#include "../../include/manatee_gpu.h"
#include "kernels_fletcher.cuh"
#include "kernels_lz4.cuh"
#include "kernels_lz4hc.cuh"
#include "kernels_codec.cuh"
#include "kernels_index.cuh"
#include "kernels_block.cuh"
#include "kernels_sha256.cuh"
#include "kernels_sha512.cuh"
#include "kernels_frames.cuh"
#include "kernels_inflate.cuh"
#include "kernels_deflate.cuh"

namespace mtz {

// block-check verdicts not yet folded into the handle: those of deferred batches wait for
// mtz_dev_finish*, where the stream verdict of the same records surfaces
struct BlockPending {
	BlockResult r{};
	uint64_t obj = 0, off = 0;    // drr_object / drr_offset of record r.first_bad
	uint8_t ctype = 0;            // ... and its drr_checksumtype
	BlockPending() { r.first_bad = r.first_frame_miss = ~0ull; }
	void clear() { *this = BlockPending(); }
};

// The counters of `r` added to those of the same names in `d` (a BlockResult or mtz_block_stats),
// and the first frame miss of both kept.
template <class Dst> static void block_add(Dst &d, const BlockResult &r)
{
	d.logical_ok += r.logical_ok; d.frame_ok += r.frame_ok; d.frame_miss += r.frame_miss; d.skipped += r.skipped;
	d.sha256 += r.sha256; d.sha512 += r.sha512;
	d.frames_encoded += r.frames_encoded; d.lzjb_encoded += r.lzjb_encoded; d.zle_encoded += r.zle_encoded;
	d.logical_checked += r.logical_checked;
	d.first_frame_miss = d.first_frame_miss < r.first_frame_miss ? d.first_frame_miss : r.first_frame_miss;
}

// device scratch of one codec batch (modes COMPRESS / DECOMPRESS / RECOMPRESS); in VERIFY with
// MTZ_FLAG_BLOCK_FRAMES / _LZJB the encoders' jobs, scratch and frame sums of the block check (enc, d_enc,
// osums, k3_skip); in the codec modes with MTZ_FLAG_BLOCK_LOGICAL the jobs, sums and encoder scratch of the
// block check's own (chk, chk_sums, d_chk, chk_pos): enc, d_enc and osums are K3's, k_assemble's and the
// output K1's there
struct CodecBufs {
	size_t rec_cap = 0, scratch_cap = 0;
	CodecRec *cr = nullptr;
	uint64_t *vals = nullptr, *offs = nullptr, *out_offs = nullptr;
	mtz_job *dec = nullptr, *enc = nullptr;
	mtz_job *dec_gz = nullptr;                          // DECOMPRESS with MTZ_FLAG_GZIP_WIRE: k_inflate's jobs (k_plan_jobs)
	mtz_job *gz = nullptr;                              // COMPRESS with MTZ_FLAG_GZIP_ENCODE: k_deflate_from_lz4's verdicts
	uint8_t *d_gz = nullptr;                            // ... and its zlib frames, at d_enc's slot offsets
	mtz_rec *out_recs = nullptr;
	RecSums *osums = nullptr;
	StampStep *steps = nullptr;                         // per-record transitions of the stamp chain
	uint8_t *d_logical = nullptr, *d_enc = nullptr;
	uint32_t *seq_n = nullptr, *cert = nullptr;         // RECOMPRESS certificate: K2's parse sizes, K3c's verdicts
	uint32_t *k3_skip = nullptr;                        // VERIFY with BLOCK_FRAMES and BLOCK_LZJB: K3 leaves these jobs
	uint32_t *hc_tab = nullptr;                         // COMPRESS with MTZ_FLAG_LZ4_HC: K3h's hash tables (hc_tab_bytes)
	mtz_job *chk = nullptr;                             // BLOCK_LOGICAL: k_logical_plan's jobs
	RecSums *chk_sums = nullptr;                        // ... and the sums of their bytes
	uint8_t *d_chk = nullptr;                           // ... with BLOCK_LZJB: the slots of the lzjb / zle frames
	unsigned long long *chk_pos = nullptr;              // ... and the running slot offset
	CodecResult *d_cres = nullptr, *h_cres = nullptr;   // h_: pinned
	ScanResult *d_ores = nullptr, *h_ores = nullptr;    // output-chain result
	uint64_t *d_outpos = nullptr;                       // running output offset (device)
	size_t avg_out_rec = 128u << 10;                    // K1 lane-group choice for the output records
};

// One GPU of the handle's device group.  Batch b of the stream runs on devs[b % G] (record-index
// partition, SURVEY.md 8e); the running checksums hop from device to device with the batches.
struct DevCtx {
	int device = 0, sm_count = 0;
	Ck4 *d_carry_in = nullptr;     // running checksum of the INPUT stream (valid on the device of the last batch)
	Ck4 *d_carry_out = nullptr;    // ... of the OUTPUT stream (codec modes)
	// fan-out (library-owned NCCL communicator over the group, one rank per device)
	ncclComm_t comm = nullptr;
	cudaStream_t fan_st = nullptr;                   // collectives + egress D2H of this device
	uint8_t *fan_buf[2] = { nullptr, nullptr };      // receive side of the broadcast (double buffered)
	size_t fan_cap = 0;
	std::vector<cudaEvent_t> ev_pool;                // egress piece events (device bound)
};

struct Slot {
	int di = 0;                   // index into mtz_handle::devs
	uint64_t seq = 0;             // stream-wide batch number of the batch in the slot
	int egress_left = 0;          // consumers that have not finished reading the slot's output
	cudaEvent_t ev_scan = nullptr;   // running checksums updated (the next batch's chain waits on it)
	cudaEvent_t ev_h2d = nullptr;    // the batch's input bytes have left the host ring
	uint8_t *d_in = nullptr;      // batch bytes (input stream slice)
	uint8_t *d_out = nullptr;     // codec modes: output slice
	size_t cap = 0, out_cap = 0;
	mtz_rec *d_recs = nullptr;
	mtz_rec *h_recs = nullptr;    // pinned staging
	size_t rec_cap = 0;
	RecSums *d_sums = nullptr;
	Part *d_tiles = nullptr;      // scan spine scratch
	ScanResult *d_res = nullptr;
	ScanResult *h_res = nullptr;  // pinned
	BlockResult *d_bres = nullptr, *h_bres = nullptr;   // MTZ_FLAG_BLOCK_CKSUM (h_: pinned)
	cudaStream_t st = nullptr;
	cudaStream_t st_k3 = nullptr;      // least-priority side stream of the LZ4 encoder (make_stream)
	cudaEvent_t ev_start = nullptr, ev_done = nullptr;
	cudaEvent_t ev_k1a = nullptr, ev_k1b = nullptr;
	cudaEvent_t ev_c0 = nullptr, ev_c1 = nullptr;     // around K2+K3
	cudaEvent_t ev_k3a = nullptr, ev_k3b = nullptr;   // around K3 alone
	bool k3_timed = false;
	bool emit_pre = false;        // COMPRESS: the slot's output is preceded by a wire preamble
	uint32_t pre_flags = 0;
	bool d2h_pending = false;     // bulk API: the slot's output copy has been issued, not awaited
	bool busy = false;
	size_t nrec = 0, bytes = 0, out_bytes = 0;
	uint64_t first_rec = 0;       // stream-wide index of the batch's first record
	uint64_t in_off = 0;          // absolute stream offset of the batch
	uint64_t writes = 0;
	CodecBufs cb;                 // per-slot codec scratch
};

struct Engine;                    // streaming state (rings + worker thread)

} // namespace mtz

struct mtz_handle {
	mtz_config cfg{};
	int device = 0;
	int sm_count = 0;
	uint32_t *k_hc_tab = nullptr;      // mtz_k_lz4hc_encode's hash tables (allocated on first use)
	uint8_t *k_gz_lz = nullptr;        // mtz_k_gzip_encode's LZ4 frames (grown on use)
	size_t k_gz_lz_cap = 0;
	std::string err;
	std::mutex err_mu;
	std::atomic<int32_t> failed{0};
	mtz_stats stats{};
	std::mutex stats_mu;

	// running checksums (device resident, updated in stream order)
	mtz::Ck4 *d_carry_in = nullptr;    // of the INPUT stream
	mtz::Ck4 *d_carry_out = nullptr;   // of the OUTPUT stream (codec modes)
	mtz::Ck4 *h_carry = nullptr;       // pinned scratch (4 entries)
	uint64_t end_ck[4] = {0, 0, 0, 0};

	std::vector<mtz::DevCtx> devs;     // devs[0].device == device
	std::vector<mtz::Slot> slots;      // slot k lives on devs[k % devs.size()]
	cudaStream_t st = nullptr;         // device-API stream (devs[0])
	int prev_scan_slot = -1;           // slot whose ev_scan the next batch's chain waits on
	bool nccl_ready = false;
	// multi-process shard exchange (mtz_comm_init): one rank per process on devs[0]
	ncclComm_t xcomm = nullptr;
	bool xcomm_owned = false;
	mtz::Ck4 *d_xbase = nullptr;       // [0] base of this round (input checksum), [1] base of the next
	int xrank = 0, xworld = 1;
	uint32_t xflags = 0;
	mtz::Part *d_xagg = nullptr, *d_xall = nullptr;
	uint64_t records_done = 0;

	// device-API / deferred-verify state: one growing table of per-record sums
	mtz::RecSums *dv_sums = nullptr;
	size_t dv_sums_cap = 0;
	mtz::Part *dv_tiles = nullptr;
	size_t dv_nrec = 0, dv_in_bytes = 0;
	uint64_t dv_first = 0;
	mtz::ScanResult *dv_res = nullptr, *dv_hres = nullptr;
	cudaStream_t dv_st = nullptr;
	cudaEvent_t dv_k1a = nullptr, dv_k1b = nullptr;
	cudaEvent_t dv_c0 = nullptr, dv_c1 = nullptr;
	std::vector<cudaEvent_t> dv_k3ev;  // pairs around the K3 launch of every sub-batch
	size_t dv_k3n = 0;
	bool dv_timed = false;

	mtz::CodecBufs dv_cb, dv_cb2;      // device-API codec scratch (sub-batched, double-buffered)
	cudaStream_t st_post = nullptr;    // layout/assemble/stamp of sub-batch k under K2/K3 of k+1
	cudaStream_t st_dec = nullptr;     // plan + K2 of sub-batch k+1 under K3 of k
	cudaEvent_t ev_dec[2] = {nullptr, nullptr};
	cudaEvent_t ev_pre[2] = {nullptr, nullptr}, ev_post[2] = {nullptr, nullptr};
	cudaEvent_t ev_reset = nullptr;        // codec_reset of this submit is done (gates st_dec / st_post)
	std::vector<mtz_rec> dv_hrecs;     // host copy of the device record table
	mtz_rec *dv_all_orecs = nullptr;   // shard mode: output table / sums of the whole submit
	mtz::RecSums *dv_all_osums = nullptr;
	mtz::StampStep *dv_all_steps = nullptr;
	size_t dv_all_cap = 0;
	uint8_t *dv_out = nullptr;

	// MTZ_FLAG_BLOCK_CKSUM: results of the device API's submit, verdicts waiting for a finish,
	// counters of the handle (under stats_mu)
	mtz::BlockResult *dv_bres = nullptr, *dv_hbres = nullptr;
	bool dv_bres_live = false;         // dv_bres holds the results of an unfinished mtz_dev_submit
	const uint8_t *dv_in = nullptr;    // ... and the batch they refer to
	const mtz_rec *dv_recs = nullptr;
	mtz::BlockPending bpend;
	mtz_block_stats bstats{};
	mtz_compressed_in_stats cstats{};  // MTZ_FLAG_COMPRESSED_IN counters (under stats_mu)

	mtz::IndexResult *d_ires = nullptr, *h_ires = nullptr;
	mtz::IndexShared *d_ishared = nullptr;

	mtz::Engine *eng = nullptr;        // created on first streaming call
	std::mutex eng_mu;
};

namespace mtz {
int32_t fail(mtz_handle *h, int32_t code, const char *fmt, ...);
int32_t fail_cuda(mtz_handle *h, cudaError_t e, const char *what);
void engine_wake_all(mtz_handle *h);
}

#define MTZ_NCCL(h, call)                                                      \
	do {                                                                       \
		ncclResult_t r__ = (call);                                             \
		if (r__ != ncclSuccess)                                                \
			return mtz::fail((h), MTZ_ECUDA, "NCCL error %d (%s) at %s", (int)r__, \
			    ncclGetErrorString(r__), #call);                               \
	} while (0)

#define MTZ_CU(h, call)                                                        \
	do {                                                                       \
		cudaError_t e__ = (call);                                              \
		if (e__ != cudaSuccess) return mtz::fail_cuda((h), e__, #call);        \
	} while (0)
