// emul_kernels.cc -- TEST INFRASTRUCTURE: C entry points that run the repository's DEVICE
// functions (compiled for the host through tests/emul/cuda_runtime.h) on one emulated warp.
#include "cuda_runtime.h"
#include "../../manatee_b200/csrc/kernels_lz4.cuh"
#include "../../manatee_b200/csrc/kernels_fletcher.cuh"
#include "../../manatee_b200/csrc/kernels_codec.cuh"
#include "../../manatee_b200/csrc/kernels_index.cuh"
#include <vector>

namespace mtz {
thread_local uint4 s_dyn[(4 * LZ4_TAB_BIG_WORDS) / 4 + 16];   // the kernels' dynamic shared memory
}

extern "C" {

// ZFS-LZ4 frame of one block through warp_zfs_lz4_compress<COMPACT>: returns psize, or lsize
// when the block is to be stored raw.  `dst` must hold lsize bytes.
uint32_t emu_zfs_lz4_compress(const uint8_t *src, uint32_t lsize, uint8_t *dst, int compact)
{
	std::vector<uint32_t> tab(LZ4_TAB_BIG_WORDS + 64, 0xdeadbeefu);     // shared memory is NOT zeroed
	uint32_t out[32];
	emu::run_warp([&](int lane) {
		out[lane] = compact ? mtz::warp_zfs_lz4_compress<true>(src, lsize, dst, tab.data(), lane)
		                    : mtz::warp_zfs_lz4_compress<false>(src, lsize, dst, tab.data(), lane);
	});
	for (int l = 1; l < 32; l++) if (out[l] != out[0]) return 0xffffffffu;    // must be warp-uniform
	return out[0];
}

// raw LZ4 block through warp_lz4_encode3 with an explicit table flavour:
// 0 = u16 x 8192 (no distance check), 1 = u32 x 4096, 2 = 17 bit x 4096 (compact)
uint32_t emu_lz4_encode_block(const uint8_t *src, uint32_t isize, uint8_t *dst, uint32_t osize, int flavour)
{
	std::vector<uint32_t> tab(LZ4_TAB_BIG_WORDS + 64, 0xdeadbeefu);
	uint32_t out[32];
	emu::run_warp([&](int lane) {
		if (flavour == 0) out[lane] = mtz::warp_lz4_encode3<mtz::TabU16, false>(src, isize, dst, osize, tab.data(), lane);
		else if (flavour == 1) out[lane] = mtz::warp_lz4_encode3<mtz::TabU32, true>(src, isize, dst, osize, tab.data(), lane);
		else out[lane] = mtz::warp_lz4_encode3<mtz::Tab17, true>(src, isize, dst, osize, tab.data(), lane);
	});
	for (int l = 1; l < 32; l++) if (out[l] != out[0]) return 0xffffffffu;
	return out[0];
}

// ZFS-LZ4 frame -> lsize bytes through warp_lz4_decode: MTZ_OK or MTZ_ECODEC
int32_t emu_zfs_lz4_decode(const uint8_t *src, uint32_t psize, uint8_t *dst, uint32_t lsize)
{
	int32_t out[32];
	emu::run_warp([&](int lane) { out[lane] = mtz::warp_lz4_decode(src, psize, dst, lsize, lane); });
	for (int l = 1; l < 32; l++) if (out[l] != out[0]) return -1000;
	return out[0];
}

// RECOMPRESS's certificate of one record, launched as the pipeline launches it: k2_lz4_decode of the
// frame with the parse by-product, then k3c_lz4_certify<flavour == 2> over `data` (lsize bytes: K2's
// output in the product) -- flavour 0 = TabU16, 1 = TabU32, 2 = Tab17 (a compact launch).
// 1 certified, 0 not, -1 flavour not one the product uses for lsize, -2 the frame does not decode,
// -3 it decodes to other bytes than `data`, -4 the certified frame length is not 4 + clen.
int32_t emu_lz4_certify(const uint8_t *frame, uint32_t psize, const uint8_t *data, uint32_t lsize, int flavour)
{
	using namespace mtz;
	const bool small = lsize < (uint32_t)LZ4_64KLIMIT;
	if ((flavour == 0) != small || flavour < 0 || flavour > 2 || (flavour == 2 && lsize > 131072u)) return -1;
	std::vector<uint8_t> dec(lsize + 64, 0xC3);
	std::vector<uint64_t> seqs(lsize / 8u + 1u, 0x0123456789abcdefull);   // the encoder's (unused) frame slot
	mtz_job jd, je;
	memset(&jd, 0, sizeof jd); memset(&je, 0, sizeof je);
	jd.src_off = (uint64_t)(uintptr_t)frame; jd.dst_off = (uint64_t)(uintptr_t)dec.data();
	jd.src_len = psize; jd.lsize = lsize;
	je.src_off = (uint64_t)(uintptr_t)data; je.dst_off = (uint64_t)(uintptr_t)seqs.data(); je.lsize = lsize;
	uint32_t seq_n = 0x5a5a5a5au, cert = 0xa5a5a5a5u;
	emu::launch(1, LZ4_THREADS, [&] { k2_lz4_decode(nullptr, nullptr, &jd, 1, &je, &seq_n); });
	if (jd.status != MTZ_OK) return -2;
	if (memcmp(dec.data(), data, lsize) != 0) return -3;
	if (flavour == 2) emu::launch(1, K3_THREADS, [&] { k3c_lz4_certify<true>(&jd, &je, &seq_n, &cert, 1); });
	else emu::launch(1, K3_THREADS, [&] { k3c_lz4_certify<false>(&jd, &je, &seq_n, &cert, 1); });
	if (cert == 0u) return 0;
	const uint32_t clen = ((uint32_t)frame[0] << 24) | ((uint32_t)frame[1] << 16) | ((uint32_t)frame[2] << 8) | frame[3];
	return cert == clen + 4u ? 1 : -4;
}

} // extern "C"

// ---- guard-page buffers: [p, p+size+slack) is accessible and the next byte is not, so a
// device function that reads or writes further than the product's buffers allow dies with
// SIGSEGV here instead of silently touching a neighbour (the CPU stand-in for memcheck).
#include <sys/mman.h>
#include <unistd.h>

extern "C" {

void *emu_guard_alloc(size_t size, size_t slack, size_t front)
{
	const size_t page = (size_t)sysconf(_SC_PAGESIZE);
	const size_t body = size + slack + front;
	const size_t npages = (body + page - 1) / page + 2;
	uint8_t *m = (uint8_t *)mmap(nullptr, npages * page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
	if (m == MAP_FAILED) return nullptr;
	uint8_t *end = m + (npages - 1) * page;                         // first inaccessible byte
	uint8_t *p = end - slack - size;
	memset(m + page, 0xA5, (size_t)(p - (m + page)));               // whatever precedes is junk, not zeros
	memset(p + size, 0x5A, slack);
	mprotect(m, page, PROT_NONE);                                   // page before
	mprotect(end, page, PROT_NONE);                                 // page after
	return p;
}

void emu_guard_free(void *p, size_t size, size_t slack, size_t front)
{
	const size_t page = (size_t)sysconf(_SC_PAGESIZE);
	const size_t body = size + slack + front;
	const size_t npages = (body + page - 1) / page + 2;
	uint8_t *end = (uint8_t *)p + size + slack;
	munmap(end - (npages - 1) * page, npages * page);
}

} // extern "C"

// ---- K1 + scan: the VERIFY pipeline's kernels, launched like launch_k1_kernel / launch_scan
// in mtz_lib.cu do (same grids' shape, same order), on the emulator.
extern "C" {

// lanes: 32 = k1_record_sums (warp per record), 16 / 8 / 4 = k1_record_sums_g<G>
int32_t emu_k1(const uint8_t *base, const mtz_rec *recs, uint32_t nrec, void *sums_out,
    uint32_t body_from, int lanes, uint32_t grid)
{
	mtz::RecSums *sums = (mtz::RecSums *)sums_out;
	if (lanes == 32) emu::launch(grid, K1_THREADS, [&] { mtz::k1_record_sums(base, recs, nrec, sums, body_from); });
	else if (lanes == 16) emu::launch(grid, K1_THREADS, [&] { mtz::k1_record_sums_g<16>(base, recs, nrec, sums, body_from); });
	else if (lanes == 8) emu::launch(grid, K1_THREADS, [&] { mtz::k1_record_sums_g<8>(base, recs, nrec, sums, body_from); });
	else if (lanes == 4) emu::launch(grid, K1_THREADS, [&] { mtz::k1_record_sums_g<4>(base, recs, nrec, sums, body_from); });
	else return -1;
	return 0;
}

uint32_t emu_recsums_size(void) { return (uint32_t)sizeof(mtz::RecSums); }

// out[0] = bad (0xffffffff none), out[1] = end_seen, out[2..5] = end_ck, out[6..9] = carry,
// out[10..14] = aggregate (n, A, B, C, D)
int32_t emu_scan_verify(const void *sums_in, uint32_t nrec, const uint64_t carry_in[4], uint64_t out[15])
{
	const mtz::RecSums *sums = (const mtz::RecSums *)sums_in;
	mtz::ScanResult res;
	memset(&res, 0, sizeof res);
	mtz::Ck4 cin = { carry_in[0], carry_in[1], carry_in[2], carry_in[3] };
	if (nrec == 0) return -1;
	const uint32_t ntiles = (nrec + SCAN_TILE - 1) / SCAN_TILE;
	std::vector<mtz::Part> tiles(ntiles + 2);
	emu::launch(ntiles, SCAN_THREADS, [&] { mtz::k_scan_tiles(sums, nrec, tiles.data()); });
	emu::launch(1, SCAN_THREADS, [&] { mtz::k_scan_spine(tiles.data(), ntiles, &res); });
	emu::launch(ntiles, SCAN_THREADS, [&] { mtz::k_scan_verify(sums, nrec, tiles.data(), &cin, &res); });
	out[0] = res.bad; out[1] = res.end_seen;
	out[2] = res.end_ck.a; out[3] = res.end_ck.b; out[4] = res.end_ck.c; out[5] = res.end_ck.d;
	out[6] = res.carry.a; out[7] = res.carry.b; out[8] = res.carry.c; out[9] = res.carry.d;
	out[10] = res.agg.n; out[11] = res.agg.a; out[12] = res.agg.b; out[13] = res.agg.c; out[14] = res.agg.d;
	return 0;
}

} // extern "C"

// ---- the re-encoding pipeline of one batch, launched in the order codec_reset /
// codec_launch_dec / codec_launch_enc / codec_launch_post (mtz_lib.cu) launch it.
extern "C" {

// res[0] = out_bytes, res[1] = bad (0xffffffff none), res[2] = n_dec, res[3] = n_enc,
// res[4..7] = end_ck of the OUTPUT stream, res[8..11] = carry_out after the batch, res[12] = end_seen
int32_t emu_codec(uint32_t mode, const uint8_t *d_in, const mtz_rec *recs, uint32_t n, uint8_t *d_out,
    const uint64_t carry_out_in[4], int k1_lanes, uint64_t res[13])
{
	using namespace mtz;
	if (n == 0) return -1;
	std::vector<CodecRec> cr(n);
	std::vector<uint64_t> vals(n), offs(n), out_offs(n);
	std::vector<mtz_job> dec(n), enc(n);
	std::vector<mtz_rec> orecs(n);
	std::vector<RecSums> osums(n);
	uint64_t scratch = 0;
	bool compact = true;
	for (uint32_t i = 0; i < n; i++) {
		if (recs[i].type == 3) {
			scratch += ((recs[i].lsize + 15u) & ~15u) + 16u;
			if (recs[i].lsize < (uint32_t)LZ4_64KLIMIT || recs[i].lsize > 131072u) compact = false;
		}
	}
	std::vector<uint8_t> d_logical(scratch + 64, 0xC3), d_enc(scratch + 64, 0x3C);
	uint64_t outpos = 0;
	CodecResult cres; memset(&cres, 0, sizeof cres); cres.bad = 0xffffffffu;
	ScanResult ores; memset(&ores, 0, sizeof ores);
	Ck4 carry = { carry_out_in[0], carry_out_in[1], carry_out_in[2], carry_out_in[3] };
	const unsigned tb = 256, gb = (n + tb - 1) / tb;

	emu::launch(gb, tb, [&] { k_plan_need(recs, n, mode, cr.data(), vals.data()); });
	emu::launch(1, XSCAN_THREADS, [&] { k_xscan_u64(vals.data(), offs.data(), n, nullptr, nullptr); });
	emu::launch(gb, tb, [&] { k_plan_jobs(d_in, recs, n, cr.data(), offs.data(), d_logical.data(), d_enc.data(), dec.data(), enc.data()); });
	const unsigned glz = (n + LZ4_WARPS - 1) / LZ4_WARPS > 3 ? 3 : (n + LZ4_WARPS - 1) / LZ4_WARPS;   // grid-stride
	if (mode != MTZ_MODE_COMPRESS)
		emu::launch(glz, LZ4_THREADS, [&] { k2_lz4_decode(nullptr, nullptr, dec.data(), n); });
	if (mode != MTZ_MODE_DECOMPRESS) {
		if (compact) emu::launch(glz, K3_THREADS, [&] { k3_lz4_encode<true>(nullptr, nullptr, enc.data(), n); });
		else emu::launch(glz, K3_THREADS, [&] { k3_lz4_encode<false>(nullptr, nullptr, enc.data(), n); });
	}
	emu::launch(gb, tb, [&] { k_layout(recs, n, cr.data(), dec.data(), enc.data(), vals.data(), &cres, 0u); });
	emu::launch(1, XSCAN_THREADS, [&] { k_xscan_u64(vals.data(), out_offs.data(), n, &outpos, &outpos); });
	const unsigned ga = (n + 7) / 8 > 4 ? 4 : (n + 7) / 8;
	emu::launch(ga, ASM_THREADS, [&] { k_assemble(d_in, recs, n, mode, cr.data(), out_offs.data(), enc.data(),
	    d_logical.data(), d_enc.data(), d_out, orecs.data()); });
	if (emu_k1(d_out, orecs.data(), n, osums.data(), 312u, k1_lanes, 2) != 0) return -2;
	std::vector<StampStep> steps(n);
	emu::launch((n + 127u) / 128u, 128, [&] { k_stamp_prep(orecs.data(), osums.data(), n, steps.data()); });
	emu::launch(1, STAMP_THREADS, [&] { k_stamp_chain(d_out, orecs.data(), osums.data(), steps.data(), n, &carry, &ores); });
	res[0] = outpos; res[1] = cres.bad; res[2] = cres.n_dec; res[3] = cres.n_enc;
	res[4] = ores.end_ck.a; res[5] = ores.end_ck.b; res[6] = ores.end_ck.c; res[7] = ores.end_ck.d;
	res[8] = carry.a; res[9] = carry.b; res[10] = carry.c; res[11] = carry.d;
	res[12] = ores.end_seen;
	return 0;
}

} // extern "C"

// ---- the GPU-side DRR parse (k_index; cooperative launch emulated with one CTA) and the
// shard carry fold
extern "C" {

// res[0] = nrec, res[1] = consumed, res[2] = status
int32_t emu_index(const uint8_t *base, uint64_t n, mtz_rec *recs, uint64_t cap, int64_t res[3])
{
	mtz::IndexResult r; memset(&r, 0, sizeof r);
	mtz::IndexShared sh; memset(&sh, 0xff, sizeof sh);
	emu::launch(1, INDEX_THREADS, [&] { mtz::k_index(base, n, recs, cap, &r, &sh); });
	res[0] = (int64_t)r.nrec; res[1] = (int64_t)r.consumed; res[2] = (int64_t)r.status;
	return 0;
}

// aggs = world x (n, A, B, C, D); carry of shard `rank` = fold of the earlier aggregates
int32_t emu_fold_carry(const uint64_t *aggs, uint32_t rank, uint64_t carry[4])
{
	mtz::Ck4 c = { 0, 0, 0, 0 };
	emu::launch(1, 1, [&] { mtz::k_fold_carry((const mtz::Part *)aggs, rank, &c); });
	carry[0] = c.a; carry[1] = c.b; carry[2] = c.c; carry[3] = c.d;
	return 0;
}

} // extern "C"

// number of barrier waits executed so far (every *_sync intrinsic is 1-2 of them per lane):
// a rough count of warp-synchronous steps, used to compare formulations offline
extern "C" unsigned long long emu_syncs(void) { return emu::syncs(); }
