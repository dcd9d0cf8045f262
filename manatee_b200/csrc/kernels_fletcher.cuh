// kernels_fletcher.cuh -- K1 (per-record Fletcher-4 sums) and the record scan that
// turns them into the running stream checksum and verifies every embedded
// drr_checksum / DRR_END checksum.
//
// Stream semantics restated from illumos dmu_send.c dump_record() /
// dmu_recv.c receive_read_record() ([EXTERNAL], SURVEY.md App. A.2): the
// reference's own code only pipes these bytes (lib/backupSender.js:179,
// lib/zfsClient.js:826).
#pragma once
#include "fletcher.cuh"
#include "../../include/manatee_gpu.h"

namespace mtz {

#define DRR_HDR    312u
#define DRR_CKOFF  280u
#define DRR_BEGIN_T 0u
#define DRR_WRITE_T 3u
#define DRR_END_T   5u

struct RecSums {         // 144 B per record: everything the scan needs, so the
	Ck4 head;            //   stream bytes can be recycled before verification
	Ck4 body;            // header[0,280) sums; body sums (see body_from)
	Ck4 emb;             // header bytes 280..311 as found in the input
	Ck4 aux;             // header bytes 8..39 (drr_end.drr_checksum for END)
	uint64_t nbody;      // words in body
	uint32_t type;       // drr_type
	uint32_t pad;
};

struct ScanResult {      // lives in device memory, mirrored to pinned host
	Part agg;            // aggregate of the batch's record bytes
	Ck4 carry;           // running checksum after the batch
	Ck4 end_ck;          // running checksum before DRR_END, if seen
	uint32_t bad;        // first failing record index in batch, 0xffffffff none
	uint32_t status;     // 0 ok, else -MTZ_E*
	uint32_t end_seen;
	uint32_t pad;
};

__device__ __forceinline__ Ck4 load_ck(const uint8_t *p)   // 8-byte aligned
{
	const uint64_t *q = reinterpret_cast<const uint64_t *>(p);
	Ck4 r = { q[0], q[1], q[2], q[3] };
	return r;
}

#define K1_THREADS 128
#define K1_WARPS   (K1_THREADS / 32)
#ifndef K1_MINBLOCKS
#define K1_MINBLOCKS 4
#endif

// One WARP per record (grid-stride).  A 128 KiB record is 257 rows of 512 B:
// the warp streams them with K1_UNROLL (12) LDG.128 in flight per lane, so the
// per-call basis conversion and the warp reduction are paid once per record.
// 4 CTAs/SM x 12 loads in flight fit 126 registers without spills.
// body_from = 280 (VERIFY: checksum field + payload) or 312 (payload only).
__global__ void __launch_bounds__(K1_THREADS, K1_MINBLOCKS)
k1_record_sums(const uint8_t *__restrict__ base, const mtz_rec *__restrict__ recs,
    uint32_t nrec, RecSums *__restrict__ out, uint32_t body_from)
{
	const int lane = threadIdx.x & 31;
	const uint32_t gw = blockIdx.x * K1_WARPS + (threadIdx.x >> 5);
	const uint32_t nw = gridDim.x * K1_WARPS;

	for (uint32_t r = gw; r < nrec; r += nw) {
		const mtz_rec rec = recs[r];
		const uint8_t *hdr = base + rec.off;
		const uint8_t *body = hdr + body_from;
		const uint32_t nwords = (DRR_HDR - body_from + rec.payload) >> 2;

		const Ck4 h = warp_fletcher(hdr, DRR_CKOFF / 4u, lane);

		// chunks of <= MTZ_K1_MAX_ROWS rows (T3(row) must fit 32 bits); chunk
		// boundaries sit on 512 B rows so only the first chunk has a head skip
		const uint32_t head = (uint32_t)(((uintptr_t)body & 511u) >> 2);
		const uint32_t first = min(nwords, MTZ_K1_MAX_ROWS * 128u - head);
		Ck4 acc = { 0, 0, 0, 0 };
		for (uint32_t w0 = 0; w0 < nwords;) {
			const uint32_t w1 = (w0 == 0u) ? first : min(nwords, w0 + MTZ_K1_MAX_ROWS * 128u);
			Ck4 p = warp_fletcher(body + 4ull * w0, w1 - w0, lane);
			if (w1 != nwords) p = shift_zeros(p, (uint64_t)(nwords - w1));
			acc.a += p.a; acc.b += p.b; acc.c += p.c; acc.d += p.d;
			w0 = w1;
		}
		if (lane == 0) {
			RecSums o;
			o.head = h; o.body = acc; o.nbody = nwords; o.pad = 0;
			o.type = rec.type;
			o.emb = load_ck(hdr + DRR_CKOFF);
			o.aux = load_ck(hdr + 8);
			out[r] = o;
		}
	}
}

// Small-record form: G lanes per record, 32/G records per warp.  Chosen by the host
// from the batch's average record size (a 128 KiB stream keeps G = 32).
template <int G>
__global__ void __launch_bounds__(K1_THREADS, K1_MINBLOCKS)
k1_record_sums_g(const uint8_t *__restrict__ base, const mtz_rec *__restrict__ recs,
    uint32_t nrec, RecSums *__restrict__ out, uint32_t body_from)
{
	constexpr uint32_t GPW = 32u / G;                      // groups per warp
	const int lane = threadIdx.x & 31;
	const int gl = lane & (G - 1);
	const uint32_t gid = (blockIdx.x * K1_WARPS + (threadIdx.x >> 5)) * GPW + (uint32_t)(lane / G);
	const uint32_t ngroups = gridDim.x * K1_WARPS * GPW;
	// all lanes of a warp iterate together (shuffles inside): pad the trip count
	const uint32_t iters = (nrec + ngroups - 1u) / ngroups;
	for (uint32_t it = 0; it < iters; it++) {
		const uint32_t r = gid + it * ngroups;
		const bool live = r < nrec;
		mtz_rec rec; rec.off = 0; rec.payload = 0; rec.type = 0; rec.lsize = 0; rec.comp = 0; rec.resv = 0;
		if (live) rec = recs[r];
		const uint8_t *hdr = base + rec.off;
		const uint8_t *body = hdr + body_from;
		const uint32_t nwords = live ? ((DRR_HDR - body_from + rec.payload) >> 2) : 0u;
		Ck4 h = { 0, 0, 0, 0 };
		if (live) h = group_head70<G>(hdr, gl); else (void)group_head70<G>(base, gl);
		// chunks of <= MTZ_K1_MAX_ROWS rows of 16*G bytes
		constexpr uint32_t RW = 4u * G;
		const uint32_t headw = (uint32_t)(((uintptr_t)body & (16u * G - 1u)) >> 2);
		const uint32_t first = min(nwords, MTZ_K1_MAX_ROWS * RW - headw);
		Ck4 acc = { 0, 0, 0, 0 };
		uint32_t w0 = 0;
		// every group runs the same number of group_fletcher calls as the slowest one
		const uint32_t my_chunks = (nwords == 0u) ? 1u : 1u + (nwords - first + MTZ_K1_MAX_ROWS * RW - 1u) / (MTZ_K1_MAX_ROWS * RW);
		uint32_t max_chunks = my_chunks;
#pragma unroll
		for (int mk = 16; mk > 0; mk >>= 1) max_chunks = max(max_chunks, __shfl_xor_sync(0xffffffffu, max_chunks, mk));
		for (uint32_t c = 0; c < max_chunks; c++) {
			const uint32_t w1 = (w0 >= nwords) ? nwords : ((c == 0u) ? first : min(nwords, w0 + MTZ_K1_MAX_ROWS * RW));
			Ck4 p = group_fletcher<G>(body + 4ull * w0, w1 - w0, gl);
			if (w1 != nwords) p = shift_zeros(p, (uint64_t)(nwords - w1));
			acc.a += p.a; acc.b += p.b; acc.c += p.c; acc.d += p.d;
			w0 = w1;
		}
		if (live && gl == 0) {
			RecSums o;
			o.head = h; o.body = acc; o.nbody = nwords; o.pad = 0;
			o.type = rec.type;
			o.emb = load_ck(hdr + DRR_CKOFF);
			o.aux = load_ck(hdr + 8);
			out[r] = o;
		}
	}
}

// ---------------------------------------------------------------------------
// Record scan.  In VERIFY the per-record transform of the running checksum is
// affine (the bytes are given), so a batch is a segmented prefix scan under
// `concat` (segments restart at DRR_BEGIN).  Three small kernels:
//   S1  tile aggregates            (grid = tiles, SCAN_TILE records per CTA)
//   S2  scan of tile aggregates    (1 CTA) -> exclusive tile prefixes, batch agg
//   S3  per-tile rescan with the carry, verify embedded/END checksums
// ---------------------------------------------------------------------------
#define SCAN_THREADS 256
#define SCAN_TILE    SCAN_THREADS          // one record per thread

__device__ __forceinline__ Part part_shfl_up(const Part &p, int delta)
{
	Part r;
	r.n = __shfl_up_sync(0xffffffffu, (unsigned long long)p.n, delta);
	r.a = __shfl_up_sync(0xffffffffu, (unsigned long long)p.a, delta);
	r.b = __shfl_up_sync(0xffffffffu, (unsigned long long)p.b, delta);
	r.c = __shfl_up_sync(0xffffffffu, (unsigned long long)p.c, delta);
	r.d = __shfl_up_sync(0xffffffffu, (unsigned long long)p.d, delta);
	return r;
}

__device__ __forceinline__ Part rec_part(const RecSums &s)
{
	Part h = { DRR_CKOFF / 4u, s.head.a, s.head.b, s.head.c, s.head.d };
	Part b = { s.nbody, s.body.a, s.body.b, s.body.c, s.body.d };
	Part r = concat(h, b);
	if (s.type == DRR_BEGIN_T) r.n |= PART_RESET;   // checksum restarts at BEGIN
	return r;
}

__device__ __forceinline__ bool ck_eq(const Ck4 &x, const Ck4 &y)
{
	return x.a == y.a && x.b == y.b && x.c == y.c && x.d == y.d;
}

__device__ __forceinline__ bool ck_zero(const Ck4 &x)
{
	return (x.a | x.b | x.c | x.d) == 0;
}

// CTA-wide scan of one Part per thread; returns the exclusive prefix of this
// thread and (in *total, valid for every thread) the CTA aggregate.
template <int THREADS>
__device__ __forceinline__ Part block_exclusive(const Part &mine, Part *s_warp, Part *total)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	Part inc = mine;
#pragma unroll
	for (int d = 1; d < 32; d <<= 1) {
		Part up = part_shfl_up(inc, d);
		if (lane >= d) inc = concat(up, inc);
	}
	if (lane == 31) s_warp[warp] = inc;
	__syncthreads();
	if (warp == 0) {
		Part w = { 0, 0, 0, 0, 0 };
		if (lane < THREADS / 32) w = s_warp[lane];
#pragma unroll
		for (int d = 1; d < 32; d <<= 1) {
			Part up = part_shfl_up(w, d);
			if (lane >= d) w = concat(up, w);
		}
		if (lane < THREADS / 32) s_warp[lane] = w;     // inclusive over warps
	}
	__syncthreads();
	Part excl = { 0, 0, 0, 0, 0 };
	if (warp > 0) excl = s_warp[warp - 1];
	Part up = part_shfl_up(inc, 1);
	if (lane > 0) excl = concat(excl, up);
	*total = s_warp[THREADS / 32 - 1];
	return excl;
}

__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_tiles(const RecSums *__restrict__ sums, uint32_t nrec, Part *__restrict__ tile_agg)
{
	__shared__ Part s_warp[SCAN_THREADS / 32];
	const uint32_t r = blockIdx.x * SCAN_TILE + threadIdx.x;
	Part mine = { 0, 0, 0, 0, 0 };
	if (r < nrec) mine = rec_part(sums[r]);
	Part total;
	(void)block_exclusive<SCAN_THREADS>(mine, s_warp, &total);
	if (threadIdx.x == 0) tile_agg[blockIdx.x] = total;
}

// single CTA: exclusive scan over the tile aggregates (looped in CTA-size steps)
__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_spine(Part *__restrict__ tile_agg, uint32_t ntiles, ScanResult *__restrict__ res)
{
	__shared__ Part s_warp[SCAN_THREADS / 32];
	Part running = { 0, 0, 0, 0, 0 };
	for (uint32_t t0 = 0; t0 < ntiles; t0 += SCAN_THREADS) {
		const uint32_t t = t0 + threadIdx.x;
		Part mine = { 0, 0, 0, 0, 0 };
		if (t < ntiles) mine = tile_agg[t];
		Part total;
		Part excl = block_exclusive<SCAN_THREADS>(mine, s_warp, &total);
		if (t < ntiles) tile_agg[t] = concat(running, excl);    // exclusive prefix
		running = concat(running, total);
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		res->agg = running;
		res->bad = 0xffffffffu;
	}
}

__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_verify(const RecSums *__restrict__ sums, uint32_t nrec,
    const Part *__restrict__ tile_prefix, const Ck4 *__restrict__ carry_in,
    ScanResult *__restrict__ res)
{
	__shared__ Part s_warp[SCAN_THREADS / 32];
	const uint32_t r = blockIdx.x * SCAN_TILE + threadIdx.x;
	Part mine = { 0, 0, 0, 0, 0 };
	RecSums rs;
	rs.type = 0xffffffffu;
	if (r < nrec) { rs = sums[r]; mine = rec_part(rs); }
	Part total;
	Part excl = block_exclusive<SCAN_THREADS>(mine, s_warp, &total);
	if (r >= nrec) return;
	Ck4 s = apply(apply(*carry_in, tile_prefix[blockIdx.x]), excl);
	bool bad = false;
	if (rs.type == DRR_BEGIN_T) s.a = s.b = s.c = s.d = 0;
	if (rs.type == DRR_END_T) {
		if (!ck_eq(rs.aux, s)) bad = true;
		res->end_ck = s;
		res->end_seen = 1;
	}
	Part h = { DRR_CKOFF / 4u, rs.head.a, rs.head.b, rs.head.c, rs.head.d };
	Ck4 mid = apply(s, h);
	if (rs.type != DRR_BEGIN_T && !ck_zero(rs.emb) && !ck_eq(rs.emb, mid)) bad = true;
	if (bad) atomicMin(&res->bad, r);
	if (r == nrec - 1u) {
		Part b = { rs.nbody, rs.body.a, rs.body.b, rs.body.c, rs.body.d };
		res->carry = apply(mid, b);
	}
}

// carry-in of shard `rank` = fold of the aggregates of all earlier shards (device-side
// twin of manatee_b200/shard.py::carry_before)
// `base` (may be null = zero) is the running checksum in front of aggs[0]; `next_base` (may be
// null) receives the one behind aggs[world-1] -- the base of the next round when the ranks take
// the stream's chunks round-robin
__global__ void k_fold_carry(const Part *__restrict__ aggs, uint32_t rank, Ck4 *__restrict__ carry,
    const Ck4 *__restrict__ base = nullptr, uint32_t world = 0, Ck4 *__restrict__ next_base = nullptr)
{
	Ck4 s = { 0, 0, 0, 0 };
	if (base != nullptr) s = *base;
	for (uint32_t r = 0; r < rank; r++) s = apply(s, aggs[r]);
	*carry = s;
	if (next_base != nullptr) {
		for (uint32_t r = rank; r < world; r++) s = apply(s, aggs[r]);
		*next_base = s;
	}
}

} // namespace mtz
