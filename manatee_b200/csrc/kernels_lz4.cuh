// kernels_lz4.cuh -- K2 (ZFS-LZ4 decode) and K3 (ZFS-LZ4 encode), sm_90a.
//
// Byte/integer work, no tensor cores.  The codec these kernels restate runs
// today inside the `zfs` children the reference spawns (`zfs send` at
// lib/backupSender.js:177 when given -c, `zfs recv` at lib/zfsClient.js:793):
// illumos lz4.c, [EXTERNAL], SURVEY.md App. A.3.  Frame = BE32 clen | LZ4 block
// | zero pad to 512 B.  One warp owns one record: the LZ4 sequence chain is
// serial by format, parallelism comes from (a) thousands of records in flight
// and (b) the 32 lanes of the warp co-operating inside every sequence.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>
#ifdef LZ4_PROF
#include <cstdio>
#endif
#include "../../include/manatee_gpu.h"

namespace mtz {

#define LZ4_MINMATCH     4
#define LZ4_LASTLITERALS 5
#define LZ4_MFLIMIT      12
#define LZ4_MINLENGTH    13
#define LZ4_MAXDIST      65535
#define LZ4_64KLIMIT     ((1 << 16) + (LZ4_MFLIMIT - 1))
#define LZ4_SKIPSTRENGTH 6

__device__ __forceinline__ uint32_t ld_u8(const uint8_t *p) { return *p; }

// --------------------------------------------------------------- K2 decode --
// status: 0 ok, else -MTZ_ECODEC.  All lanes run the same control flow; `ip`,
// `op` and every parsed field are warp-uniform.
//
// Optional by-product (RECOMPRESS, see warp_lz4_certify): the parse of the block as a table of
// sequences, one u64 per match -- bits 0..23 the decoded position where the match starts (= anchor
// + literal length), 24..39 the offset, 40..63 the match length -- and their count in *seq_n
// (LZ4_SEQ_NONE when the table overflowed `seq_cap` or the block is not in the encoder's normal
// form: the closing literals-only token must have a zero low nibble).
#define LZ4_SEQ_NONE 0xffffffffu
__device__ __forceinline__ uint64_t lz4_seq_pack(uint32_t m, uint32_t off, uint32_t ml)
{
	return (uint64_t)m | ((uint64_t)off << 24) | ((uint64_t)ml << 40);
}

__device__ __forceinline__ int32_t warp_lz4_decode(const uint8_t *__restrict__ src,
    uint32_t psize, uint8_t *__restrict__ dst, uint32_t lsize, int lane,
    uint64_t *__restrict__ seq = nullptr, uint32_t seq_cap = 0, uint32_t *seq_n = nullptr)
{
	uint32_t ns = 0;
	if (seq_n != nullptr && lane == 0) *seq_n = LZ4_SEQ_NONE;
	if (psize < 4u) return MTZ_ECODEC;
	const uint32_t clen = (ld_u8(src) << 24) | (ld_u8(src + 1) << 16) | (ld_u8(src + 2) << 8) | ld_u8(src + 3);
	if ((uint64_t)clen + 4u > psize || clen == 0u) return MTZ_ECODEC;
	const uint8_t *in = src + 4;
	uint32_t ip = 0, op = 0;
	const uint32_t iend = clen;

	for (;;) {
		if (ip >= iend) return MTZ_ECODEC;
		const uint32_t tok = ld_u8(in + ip++);
		uint32_t len = tok >> 4;
		if (len == 15u) {
			uint32_t s;
			do {
				if (ip >= iend) return MTZ_ECODEC;
				s = ld_u8(in + ip++);
				len += s;
			} while (s == 255u);
		}
		if (len > iend - ip || len > lsize - op) return MTZ_ECODEC;
		if ((uint32_t)lane < len) dst[op + (uint32_t)lane] = in[ip + (uint32_t)lane];
		if (len > 32u)
			for (uint32_t i = 32u + (uint32_t)lane; i < len; i += 32u) dst[op + i] = in[ip + i];
		ip += len; op += len;
		if (ip == iend) {                              // last sequence: literals only
			if ((tok & 15u) != 0u) ns = LZ4_SEQ_NONE;
			break;
		}

		if (iend - ip < 2u) return MTZ_ECODEC;
		const uint32_t off = ld_u8(in + ip) | (ld_u8(in + ip + 1) << 8);
		ip += 2;
		if (off == 0u || off > op) return MTZ_ECODEC;
		uint32_t ml = tok & 15u;
		if (ml == 15u) {
			uint32_t s;
			do {
				if (ip >= iend) return MTZ_ECODEC;
				s = ld_u8(in + ip++);
				ml += s;
			} while (s == 255u);
		}
		ml += LZ4_MINMATCH;
		if (ml > lsize - op) return MTZ_ECODEC;
		if (seq != nullptr) {
			if (ns < seq_cap && lane == 0) seq[ns] = lz4_seq_pack(op, off, ml);
			ns++;
		}
		__syncwarp();                                  // earlier stores -> these loads
		const uint8_t *ref = dst + (op - off);
		if (off >= ml) {
			if ((uint32_t)lane < ml) dst[op + (uint32_t)lane] = ref[lane];
			if (ml > 32u)
				for (uint32_t i = 32u + (uint32_t)lane; i < ml; i += 32u) dst[op + i] = ref[i];
		} else {
			// overlapping match: the source is periodic with period `off`; i % off is kept
			// incrementally (one division per match instead of one per byte)
			uint32_t r = (uint32_t)lane % off;
			const uint32_t stp = 32u % off;
			for (uint32_t i = (uint32_t)lane; i < ml; i += 32u) {
				dst[op + i] = ref[r];
				r += stp;
				if (r >= off) r -= off;
			}
		}
		op += ml;
	}
	__syncwarp();
	if (op != lsize) return MTZ_ECODEC;
	if (seq_n != nullptr && lane == 0 && ns <= seq_cap) *seq_n = ns;     // (LZ4_SEQ_NONE > any cap)
	return MTZ_OK;
}

#define LZ4_THREADS 128
#define LZ4_WARPS   (LZ4_THREADS / 32)

__global__ void __launch_bounds__(LZ4_THREADS)
k2_lz4_decode(const uint8_t *__restrict__ src_base, uint8_t *__restrict__ dst_base,
    mtz_job *__restrict__ jobs, uint32_t njobs,
    const mtz_job *__restrict__ seq_jobs = nullptr, uint32_t *__restrict__ seq_n = nullptr)
{
	const int lane = threadIdx.x & 31;
	const uint32_t gw = blockIdx.x * LZ4_WARPS + (threadIdx.x >> 5);
	const uint32_t nw = gridDim.x * LZ4_WARPS;
	for (uint32_t j = gw; j < njobs; j += nw) {
		const mtz_job job = jobs[j];
		if (job.lsize == 0u) continue;                 // not a decode job (pipeline: 1 job slot per record)
		// RECOMPRESS: the parse goes into the record's (still unused) frame slot of the encoder
		uint64_t *seq = nullptr;
		if (seq_jobs != nullptr) seq = reinterpret_cast<uint64_t *>((uintptr_t)seq_jobs[j].dst_off);
		const int32_t st = warp_lz4_decode(src_base + job.src_off, job.src_len,
		    dst_base + job.dst_off, job.lsize, lane, seq, seq ? (job.lsize >> 3) : 0u,
		    seq ? seq_n + j : nullptr);
		if (lane == 0) {
			jobs[j].status = st;
			jobs[j].out_len = (st == MTZ_OK) ? job.lsize : 0u;
		}
	}
}


// --------------------------------------------------------------- K3 encode --
// Bit-exact warp-parallel form of the serial greedy matcher (oracle:
// oracle/lz4_zfs.c lz4_encode).  The serial search examines positions
// p_0, p_1, ... with step (67+a)>>6 at attempt a, reading and then updating
// hash-table slot hash(p_a) each time.  A round evaluates 32 consecutive
// attempts at once: lane L takes attempt a0+L, sees the table as the serial
// code would (older lanes of the same round with an equal hash are forwarded
// through __match_any_sync), the first lane whose candidate matches wins, and
// only lanes up to the winner commit their table updates.

__device__ __forceinline__ uint32_t ld32u(const uint8_t *p)
{
	const uintptr_t a = (uintptr_t)p;
	const uint32_t *w = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
	const uint32_t sh = (uint32_t)(a & 3u) * 8u;
	return __funnelshift_r(__ldg(w), __ldg(w + 1), sh);       // source is read-only while encoding
}

// unaligned u32 at byte offset x of a 4-byte aligned base (32-bit index math only)
__device__ __forceinline__ uint32_t ld32x(const uint32_t *__restrict__ base4, uint32_t x)
{
	const uint32_t i = x >> 2;
	return __funnelshift_r(__ldg(base4 + i), __ldg(base4 + i + 1u), (x & 3u) * 8u);
}

// sum_{i<x} ((67+i)>>6): distance covered by the first x search attempts
__device__ __forceinline__ uint32_t skip_dist(uint32_t x)
{
	const uint32_t T = 67u + x, q = T >> 6, r = T & 63u;
	return 64u * (q * (q - 1u) / 2u) + q * r - 3u;
}

// ---- hash tables (shared memory, one per warp) ----------------------------
struct TabU32 {                                 // 4096 x u32: any block size
	uint32_t *t;
	static constexpr int LOG = 12;
	__device__ __forceinline__ void clear(int lane) const {
		for (int i = lane; i < 4096; i += 32) t[i] = 0;
	}
	__device__ __forceinline__ uint32_t get(uint32_t h) const { return t[h]; }
	__device__ __forceinline__ void set(uint32_t h, uint32_t v) const { t[h] = v; }
	__device__ __forceinline__ void set_from(uint32_t h, uint32_t v, uint32_t) const { t[h] = v; }
	// slot used as a scratch mark while its value is held in a register (see search)
	__device__ __forceinline__ void tag(uint32_t h, uint32_t v) const { t[h] = v; }
	__device__ __forceinline__ uint32_t tagval(uint32_t h) const { return t[h]; }
	__device__ __forceinline__ void untag(uint32_t h, uint32_t old) const { t[h] = old; }
};
struct TabU16 {                                 // 8192 x u16: blocks below 64 KiB + 11
	uint32_t *t;
	static constexpr int LOG = 13;
	__device__ __forceinline__ void clear(int lane) const {
		for (int i = lane; i < 4096; i += 32) t[i] = 0;
	}
	__device__ __forceinline__ uint32_t get(uint32_t h) const { return reinterpret_cast<uint16_t *>(t)[h]; }
	__device__ __forceinline__ void set(uint32_t h, uint32_t v) const { reinterpret_cast<uint16_t *>(t)[h] = (uint16_t)v; }
	__device__ __forceinline__ void set_from(uint32_t h, uint32_t v, uint32_t) const { reinterpret_cast<uint16_t *>(t)[h] = (uint16_t)v; }
	__device__ __forceinline__ void tag(uint32_t h, uint32_t v) const { reinterpret_cast<uint16_t *>(t)[h] = (uint16_t)v; }
	__device__ __forceinline__ uint32_t tagval(uint32_t h) const { return reinterpret_cast<uint16_t *>(t)[h]; }
	__device__ __forceinline__ void untag(uint32_t h, uint32_t old) const { reinterpret_cast<uint16_t *>(t)[h] = (uint16_t)old; }
};
struct Tab17 {                                  // 4096 x 17 bit: blocks up to 128 KiB in 8.5 KiB
	uint32_t *t;                                // [0,2048) u16 pairs, [2048,2176) bit 16 of each slot
	static constexpr int LOG = 12;
	__device__ __forceinline__ void clear(int lane) const {
		for (int i = lane; i < 2176; i += 32) t[i] = 0;
	}
	__device__ __forceinline__ uint32_t get(uint32_t h) const {
		const uint32_t lo = reinterpret_cast<uint16_t *>(t)[h];
		const uint32_t hi = (t[2048u + (h >> 5)] >> (h & 31u)) & 1u;
		return lo | (hi << 16);
	}
	// bit 16 of a slot flips at most once per record (positions cross 64 KiB once): only
	// then is the ~100-cycle shared-memory atomic paid
	__device__ __forceinline__ void set_from(uint32_t h, uint32_t v, uint32_t old) const {
		reinterpret_cast<uint16_t *>(t)[h] = (uint16_t)v;
		if (((v ^ old) >> 16) & 1u) atomicXor(&t[2048u + (h >> 5)], 1u << (h & 31u));
	}
	__device__ __forceinline__ void set(uint32_t h, uint32_t v) const {
		const uint32_t oldhi = (t[2048u + (h >> 5)] >> (h & 31u)) & 1u;
		set_from(h, v, oldhi << 16);
	}
	// only the low half is used as the mark; bit 16 of the slot stays in the bitmap
	__device__ __forceinline__ void tag(uint32_t h, uint32_t v) const { reinterpret_cast<uint16_t *>(t)[h] = (uint16_t)v; }
	__device__ __forceinline__ uint32_t tagval(uint32_t h) const { return reinterpret_cast<uint16_t *>(t)[h]; }
	__device__ __forceinline__ void untag(uint32_t h, uint32_t old) const { reinterpret_cast<uint16_t *>(t)[h] = (uint16_t)old; }
};

#define LZ4_TAB_BIG_WORDS     4096u             // TabU32 / TabU16: 16 KiB
#define LZ4_TAB_COMPACT_WORDS 2176u             // Tab17: 8.5 KiB

// cooperative store of a 255-run length extension (value = len - 15 already)
__device__ __forceinline__ uint32_t put_len_ext(uint8_t *dst, uint32_t op, uint32_t v, int lane)
{
	const uint32_t n255 = v / 255u;
	for (uint32_t i = (uint32_t)lane; i < n255; i += 32u) dst[op + i] = 255;
	if (lane == 0) dst[op + n255] = (uint8_t)(v - n255 * 255u);
	return op + n255 + 1u;
}

// ---------------------------------------------------------------------------
// The matcher.  One LZ4 sequence costs three dependent global round trips (an
// earlier version needed seven; K3 is bound by latency chains at <= 24 warps/SM,
// not by bandwidth):
//   trip A  candidate gather of a search round (positions come preloaded)
//   trip B  catch-up bytes + first 32 literals + first match-extension round
//   trip C  follow-on probe + its extension round + next search round's positions
// The 6 bytes around the match end that the table inserts hash come out of the
// extension round's registers by shuffle.
struct ExtRound {            // one 128-byte extension round held in registers
	uint32_t wa, wb;         // words at ip0 + 4*lane and ref0 + 4*lane (0 when not loaded)
};

__device__ __forceinline__ ExtRound ext_load(const uint8_t *src, uint32_t ip0, uint32_t ref0,
    uint32_t iend, int lane)
{
	ExtRound e; e.wa = 0; e.wb = 0;
	const uint32_t o = 4u * (uint32_t)lane;
	if (ip0 + o + 4u <= iend) { e.wa = ld32u(src + ip0 + o); e.wb = ld32u(src + ref0 + o); }
	return e;
}

__device__ __forceinline__ uint32_t extract32(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t off)
{
	return (off < 4u) ? __funnelshift_r(w0, w1, off * 8u) : __funnelshift_r(w1, w2, (off - 4u) * 8u);
}

#ifdef LZ4_PROF
// clock64 phase profile (compile with -DLZ4_PROF): cycles per phase, printed by one warp
#define PROF_DECL long long pt = clock64(), p_search = 0, p_b = 0, p_ext = 0, p_post = 0; unsigned n_seq = 0, n_round = 0, n_follow = 0;
#define PROF_LAP(acc) { const long long now_ = clock64(); acc += now_ - pt; pt = now_; }
#else
#define PROF_DECL
#define PROF_LAP(acc)
#endif

template <class TAB, bool DIST>
__device__ __forceinline__ uint32_t warp_lz4_encode3(const uint8_t *__restrict__ src,
    uint32_t isize, uint8_t *__restrict__ dst, uint32_t osize, uint32_t *tabmem, int lane)
{
	constexpr int LOG = TAB::LOG;
	PROF_DECL
	const uint32_t mis = (uint32_t)((uintptr_t)src & 3u);
	const uint32_t *base4 = reinterpret_cast<const uint32_t *>(src - mis);
#define LDS32(pos) ld32x(base4, (pos) + mis)
	TAB tab; tab.t = tabmem;
	const uint32_t lanebit = 1u << lane, lower = lanebit - 1u;
	tab.clear(lane);
	__syncwarp();

	uint32_t ip = 0, anchor = 0, op = 0;
	const uint32_t iend = isize;
	if (isize >= (uint32_t)LZ4_MINLENGTH) {
		const uint32_t mflimit = iend - LZ4_MFLIMIT;
		const uint32_t matchlimit = iend - LZ4_LASTLITERALS;
		ip = 1;
		bool have_pre = false;         // vpre holds rd32(start + lane) for the next search
		uint32_t vpre = 0;
		for (;;) {
			// ------------------------------------------------ search (trip A per round)
			uint32_t ref = 0;
			bool to_tail = false;
			const uint32_t start = ip;
			for (uint32_t a0 = 0;; a0 += 32u) {
				uint32_t p, step;
				if (a0 == 0u) {                              // attempts 0..31: step 1, p = start + lane
					p = start + (uint32_t)lane; step = 1u;
				} else {
					const uint32_t a = a0 + (uint32_t)lane;
					p = start + skip_dist(a);
					step = (67u + a) >> 6;
				}
				const bool valid = (p + step <= mflimit);
				uint32_t h = 0xffffffffu - (uint32_t)lane, cand = 0, v = 0;
				if (valid) {
					v = (a0 == 0u && have_pre) ? vpre : LDS32(p);
					h = (v * 2654435761u) >> (32 - LOG);
				}
				// Do two lanes of this round hash to the same slot?  __match_any_sync answers
				// that but costs hundreds of cycles when all 32 values differ (the common
				// case; tools/micro/match_any.cu measures it).  Cheaper: every lane already holds its
				// slot's value, so mark the slots with lane ids (~100 cycles) and look back.
				uint32_t oldv = 0;
				if (valid) oldv = tab.get(h);
				__syncwarp();
				if (valid) tab.tag(h, (uint32_t)lane);
				__syncwarp();
				const bool clash = valid && (tab.tagval(h) != (uint32_t)lane);
				int F, I;
				if (!__any_sync(0xffffffffu, clash)) {
					// all slots distinct: no in-round forwarding, every lane owns its slot
					bool hit = false;
					cand = oldv;
					if (valid && (!DIST || cand + LZ4_MAXDIST >= p)) hit = (LDS32(cand) == v);
					const uint32_t hits = __ballot_sync(0xffffffffu, hit);
					const uint32_t inval = __ballot_sync(0xffffffffu, !valid);
					F = hits ? (__ffs((int)hits) - 1) : 32;
					I = inval ? (__ffs((int)inval) - 1) : 32;
					if (I < F) { to_tail = true; break; }      // table is not used after this
					if (valid) {
						if (lane <= F) tab.set_from(h, p, oldv); else tab.untag(h, oldv);
					}
				} else {
					if (valid) tab.untag(h, oldv);
					__syncwarp();
					const uint32_t all_same = __match_any_sync(0xffffffffu, h);
					const uint32_t same = all_same & lower;
					const int from = same ? (31 - __clz((int)same)) : lane;
					const uint32_t fwd = __shfl_sync(0xffffffffu, p, from);
					bool hit = false;
					if (valid) {
						cand = same ? fwd : oldv;
						if (!DIST || cand + LZ4_MAXDIST >= p) hit = (LDS32(cand) == v);
					}
					const uint32_t hits = __ballot_sync(0xffffffffu, hit);
					const uint32_t inval = __ballot_sync(0xffffffffu, !valid);
					F = hits ? (__ffs((int)hits) - 1) : 32;
					I = inval ? (__ffs((int)inval) - 1) : 32;
					if (I < F) { to_tail = true; break; }
					const uint32_t upto = (F >= 31) ? 0xffffffffu : ((2u << F) - 1u);
					const uint32_t later = all_same & ~(lanebit | lower) & upto;
					if ((lanebit & upto) && later == 0u) tab.set_from(h, p, oldv);
				}
				__syncwarp();
				if (F < 32) {
					ip = __shfl_sync(0xffffffffu, p, F);
					ref = __shfl_sync(0xffffffffu, cand, F);
					break;
				}
			}
			have_pre = false;
			PROF_LAP(p_search)
			if (to_tail) break;
#ifdef LZ4_PROF
			n_seq++;
#endif

			// ------------------------------------------------ trip B: issue everything
			// that depends only on (ip, ref) before consuming any of it
			const uint32_t k = (uint32_t)lane + 1u;
			const bool cu_ok = (ip >= anchor + k && ref >= k);
			uint32_t ca = 0, cb = 1;
			if (cu_ok) { ca = src[ip - k]; cb = src[ref - k]; }
			uint32_t lit0 = 0;
			if (anchor + (uint32_t)lane < ip) lit0 = src[anchor + (uint32_t)lane];
			ExtRound er = ext_load(src, ip, ref, iend, lane);   // lane 0 = the 4 matched bytes

			// catch up (first 32 candidates from the preloaded bytes)
			const uint32_t ip_pre = ip, ref_pre = ref;
			{
				const uint32_t ne = ~__ballot_sync(0xffffffffu, cu_ok && ca == cb);
				uint32_t n = ne ? (uint32_t)(__ffs((int)ne) - 1) : 32u;
				ip -= n; ref -= n;
				while (n == 32u) {
					bool eq = false;
					if (ip >= anchor + k && ref >= k) eq = (src[ip - k] == src[ref - k]);
					const uint32_t ne2 = ~__ballot_sync(0xffffffffu, eq);
					n = ne2 ? (uint32_t)(__ffs((int)ne2) - 1) : 32u;
					ip -= n; ref -= n;
				}
			}

			// ---------------------------------------------- literals --
			const uint32_t litlen = ip - anchor;
			uint32_t token = op++;
			if (op + litlen + (2u + 1u + LZ4_LASTLITERALS) + (litlen >> 8) > osize) return 0u;
			uint32_t tokval;
			if (litlen >= 15u) {
				tokval = 15u << 4;
				op = put_len_ext(dst, op, litlen - 15u, lane);
			} else {
				tokval = litlen << 4;
			}
			if ((uint32_t)lane < litlen) dst[op + (uint32_t)lane] = (uint8_t)lit0;
			for (uint32_t i = 32u + (uint32_t)lane; i < litlen; i += 32u) dst[op + i] = src[anchor + i];
			op += litlen;

			PROF_LAP(p_b)
			// ------------------------------- one or more back-to-back matches --
			uint32_t ext_ip = ip_pre, ext_ref = ref_pre;     // where round `er` starts
			for (;;) {
				if (lane == 0) {
					dst[op] = (uint8_t)((ip - ref) & 0xffu);
					dst[op + 1] = (uint8_t)((ip - ref) >> 8);
				}
				op += 2;
				anchor = ip + LZ4_MINMATCH;
				// extension: rounds of 128 bytes from (ext_ip, ext_ref); round 0 preloaded
				uint32_t prev31 = 0, v_end = 0, v_m2 = 0;
				for (;;) {
					const uint32_t o = 4u * (uint32_t)lane;
					const uint32_t room = (ext_ip + o < matchlimit) ? (matchlimit - ext_ip - o) : 0u;
					uint32_t n = 0;
					if (room) {
						const uint32_t x = er.wa ^ er.wb;
						n = x ? (uint32_t)((__ffs((int)x) - 1) >> 3) : 4u;
						if (n > room) n = room;
					}
					const uint32_t part = __ballot_sync(0xffffffffu, n < 4u);
					if (part) {
						const int Fp = __ffs((int)part) - 1;
						const uint32_t nf = __shfl_sync(0xffffffffu, n, Fp);
						ip = ext_ip + 4u * (uint32_t)Fp + nf;
						// bytes [ip-2, ip+4) from the registers of lanes Fp-1, Fp, Fp+1
						const uint32_t w1 = __shfl_sync(0xffffffffu, er.wa, Fp);
						uint32_t w0 = __shfl_sync(0xffffffffu, er.wa, (Fp + 31) & 31);
						uint32_t w2 = __shfl_sync(0xffffffffu, er.wa, (Fp + 1) & 31);
						if (Fp == 0) w0 = prev31;
						if (Fp == 31 && nf > 0u) w2 = (ip + 4u <= iend) ? LDS32(ext_ip + 128u) : 0u;
						v_m2 = extract32(w0, w1, w2, nf + 2u);
						v_end = extract32(w0, w1, w2, nf + 4u);
						break;
					}
					prev31 = __shfl_sync(0xffffffffu, er.wa, 31);
					ext_ip += 128u; ext_ref += 128u;
					er = ext_load(src, ext_ip, ext_ref, iend, lane);
				}
				uint32_t mlen = ip - anchor;
				if (op + (1u + LZ4_LASTLITERALS) + (mlen >> 8) > osize) return 0u;
				if (mlen >= 15u) {
					tokval += 15u;
					op = put_len_ext(dst, op, mlen - 15u, lane);
				} else {
					tokval += mlen;
				}
				if (lane == 0) dst[token] = (uint8_t)tokval;
				PROF_LAP(p_ext)

				if (ip > mflimit) { anchor = ip; to_tail = true; break; }

				// insert ip-2, then probe ip (trip C carries the probe, its extension
				// round and the next search round's positions)
				const uint32_t h2 = (v_m2 * 2654435761u) >> (32 - LOG);
				if (lane == 0) tab.set(h2, ip - 2u);
				__syncwarp();
				const uint32_t hh = (v_end * 2654435761u) >> (32 - LOG);
				const uint32_t pref = tab.get(hh);
				__syncwarp();
				if (lane == 0) tab.set_from(hh, ip, pref);
				__syncwarp();
				const uint32_t np = ip + 1u + (uint32_t)lane;          // next search, step 1
				uint32_t vn = 0;
				if (np + 1u <= mflimit) vn = LDS32(np);
				ExtRound e2 = ext_load(src, ip, pref, iend, lane);
				const bool probe_hit = (!DIST || pref + LZ4_MAXDIST >= ip) &&
				    (__shfl_sync(0xffffffffu, e2.wb, 0) == v_end);
				PROF_LAP(p_post)
				if (probe_hit) {
#ifdef LZ4_PROF
					n_follow++;
#endif
					ref = pref;
					token = op++;
					tokval = 0;
					er = e2; ext_ip = ip; ext_ref = ref;
					continue;
				}
				vpre = vn; have_pre = true;
				break;
			}
			if (to_tail) break;
			anchor = ip++;
		}
	}
	// ---------------------------------------------------- last literals --
	{
		const uint32_t last = iend - anchor;
		if (op + last + 1u + ((last + 255u - 15u) / 255u) > osize) return 0u;
		if (last >= 15u) {
			if (lane == 0) dst[op] = (uint8_t)(15u << 4);
			op = put_len_ext(dst, op + 1u, last - 15u, lane);
		} else {
			if (lane == 0) dst[op] = (uint8_t)(last << 4);
			op += 1u;
		}
		for (uint32_t i = (uint32_t)lane; i < last; i += 32u) dst[op + i] = src[anchor + i];
		op += last;
	}
#ifdef LZ4_PROF
	if (lane == 0 && blockIdx.x == 7 && (threadIdx.x >> 5) == 1 && n_seq > 100)
		printf("K3PROF seq=%u follow=%u per-seq cycles: search %lld  B(loads+catchup+literals) %lld  ext+emit %lld  post(probe) %lld  total %lld\n",
		    n_seq, n_follow, p_search / n_seq, p_b / n_seq, p_ext / n_seq, p_post / n_seq,
		    (p_search + p_b + p_ext + p_post) / n_seq);
#endif
#undef LDS32
	return op;
}

// zio_compress_data(LZ4) + 512 B sector rounding.  out_len = psize (frame
// stored at dst) or lsize (store raw: dst content is scratch).  COMPACT: the
// launch reserved only the 8.5 KiB table (every block is 64 KiB+11 .. 128 KiB).
template <bool COMPACT>
__device__ __forceinline__ uint32_t warp_zfs_lz4_compress(const uint8_t *__restrict__ src,
    uint32_t lsize, uint8_t *__restrict__ dst, uint32_t *tabmem, int lane)
{
	const uint32_t d_len = lsize - (lsize >> 3);
	if (lsize < 1024u || lsize > (16u << 20) || d_len < 4u) return lsize;
	uint32_t blk;
	if (COMPACT)
		blk = warp_lz4_encode3<Tab17, true>(src, lsize, dst + 4, d_len - 4u, tabmem, lane);
	else if (lsize < (uint32_t)LZ4_64KLIMIT)
		blk = warp_lz4_encode3<TabU16, false>(src, lsize, dst + 4, d_len - 4u, tabmem, lane);
	else
		blk = warp_lz4_encode3<TabU32, true>(src, lsize, dst + 4, d_len - 4u, tabmem, lane);
	__syncwarp();
	if (blk == 0u) return lsize;
	const uint32_t c_len = blk + 4u;
	if (c_len > d_len) return lsize;
	const uint32_t psize = (c_len + 511u) & ~511u;
	if (psize >= lsize) return lsize;
	if (lane == 0) {
		dst[0] = (uint8_t)(blk >> 24); dst[1] = (uint8_t)(blk >> 16);
		dst[2] = (uint8_t)(blk >> 8);  dst[3] = (uint8_t)blk;
	}
	for (uint32_t i = c_len + (uint32_t)lane; i < psize; i += 32u) dst[i] = 0;
	return psize;
}

// ------------------------------------------------------ K3c: the certificate --
// RECOMPRESS re-encodes what it has just decoded.  When the incoming block already IS what
// lz4_encode (oracle/lz4_zfs.c:85-208) would emit for those bytes -- every block a `zfs send -c` of an
// lz4 dataset carries, if the declared encoder is ZFS's -- the answer is the input, and PROVING that
// is far cheaper than recomputing it: the serial matcher is a chain of thousands of dependent cycles
// per sequence because every decision waits for a gather from the source; a
// replay that is TOLD the parse (K2's sequence table) knows where the hits must be and only has to
// keep the hash table honest.
//
// The proof obligation, exactly: the encoder's run on the decoded bytes D is determined by its hash
// table trajectory.  Inserted positions are strictly increasing in time (search attempts, then e-2
// and e after a match ending at e), so "the slot's content" is "the largest inserted position below
// me with my hash, else 0".  The replay executes the SAME attempts in the SAME order, 32 per round
// with the in-round forwarding of warp_lz4_encode3, under the hypothesis "the table reads a match at
// the first attempt >= m_k with offset o_k, and nowhere earlier".  Where the hypothesis says HIT it
// checks the slot arithmetically (slot == x - o_k; the bytes are equal by construction, D was
// decoded from this very parse, and o_k <= 65535); where it says MISS it checks the encoder's own
// test (distance, then 4 bytes) on a load nobody waits for (verified one round later).  A hit the
// table does not deliver at the first candidate is searched for at the following attempts (the
// matcher found the match further right and walked back: catch-up), exactly as the encoder would.
// Per match, without the table: the walk-back stops at m_k (anchor, source start or a differing
// byte), the extension stops at e_k (matchlimit or a differing byte), and the encoder's output-room
// tests, evaluated at the same output offsets, never fire.  Any violated check => not certified =>
// the record takes the serial encoder.  Certified => output frame = BE32(clen) + input block + pad.
template <class TAB>
struct TabRound {            // one round of <= 32 time-ordered table operations (lane order = time order)
	uint32_t oldv, all_same;
	bool anyclash;
};

template <class TAB>
__device__ __forceinline__ uint32_t tab_round_query(const TAB &tab, TabRound<TAB> &r, bool part,
    uint32_t h, uint32_t x, int lane)
{
	const uint32_t lanebit = 1u << lane, lower = lanebit - 1u;
	r.oldv = part ? tab.get(h) : 0u;
	__syncwarp();
	if (part) tab.tag(h, (uint32_t)lane);
	__syncwarp();
	const bool clash = part && (tab.tagval(h) != (uint32_t)lane);
	r.anyclash = __any_sync(0xffffffffu, clash);
	r.all_same = 0;
	if (!r.anyclash) return r.oldv;
	if (part) tab.untag(h, r.oldv);
	__syncwarp();
	r.all_same = __match_any_sync(0xffffffffu, h);          // non-participants carry unique fake hashes
	const uint32_t same = r.all_same & lower;
	const int from = same ? (31 - __clz((int)same)) : lane;
	const uint32_t fwd = __shfl_sync(0xffffffffu, x, from);
	return same ? fwd : r.oldv;
}

// lanes <= upto keep their insertions, the rest of the round never happened
template <class TAB>
__device__ __forceinline__ void tab_round_commit(const TAB &tab, const TabRound<TAB> &r, bool part,
    uint32_t h, uint32_t x, int upto, int lane)
{
	const uint32_t lanebit = 1u << lane, lower = lanebit - 1u;
	if (!r.anyclash) {
		if (part) {
			if (lane <= upto) tab.set_from(h, x, r.oldv); else tab.untag(h, r.oldv);
		}
	} else {
		const uint32_t uptomask = (upto >= 31) ? 0xffffffffu : ((2u << upto) - 1u);
		const uint32_t later = r.all_same & ~(lanebit | lower) & uptomask;
		if (part && (lanebit & uptomask) && later == 0u) tab.set_from(h, x, r.oldv);
	}
	__syncwarp();
}

template <class TAB, bool DIST>
__device__ __forceinline__ bool warp_lz4_certify(const uint8_t *__restrict__ src, uint32_t isize,
    const uint64_t *__restrict__ seqs, uint32_t ns, uint32_t clen, uint32_t osize,
    uint32_t *tabmem, int lane)
{
	constexpr int LOG = TAB::LOG;
	const uint32_t mis = (uint32_t)((uintptr_t)src & 3u);
	const uint32_t *base4 = reinterpret_cast<const uint32_t *>(src - mis);
#define LDS32(pos) ld32x(base4, (pos) + mis)
#define SEQ_M(s) ((uint32_t)(s) & 0xffffffu)
#define SEQ_O(s) ((uint32_t)((s) >> 24) & 0xffffu)
#define SEQ_L(s) ((uint32_t)((s) >> 40))
	const uint32_t iend = isize;
	bool bad = false;
	if (isize < (uint32_t)LZ4_MINLENGTH) {
		// the encoder goes straight to its last-literals block
		bad = (ns != 0u) || (isize + 1u + ((isize + 255u - 15u) / 255u) > osize) ||
		    (1u + (isize >= 15u ? 1u + (isize - 15u) / 255u : 0u) + isize != clen);
		return !bad;
	}
	const uint32_t mflimit = iend - LZ4_MFLIMIT;
	const uint32_t matchlimit = iend - LZ4_LASTLITERALS;

	// ---- per match, 32 at a time: catch-up stop, extension stop, output-room tests
	{
		uint32_t op = 0, prev_e = 0;
		for (uint32_t k0 = 0; k0 < ns; k0 += 32u) {
			const uint32_t k = k0 + (uint32_t)lane;
			const bool live = k < ns;
			const uint64_t s = live ? seqs[k] : 0ull;
			const uint32_t m = SEQ_M(s), o = SEQ_O(s), ml = SEQ_L(s), e = m + ml;
			uint32_t a = __shfl_up_sync(0xffffffffu, e, 1);
			if (lane == 0) a = prev_e;
			const uint32_t litlen = m - a;
			const uint32_t lb = 1u + (litlen >= 15u ? 1u + (litlen - 15u) / 255u : 0u) + litlen;
			const uint32_t mlen = ml - LZ4_MINMATCH;
			const uint32_t mb = 2u + (mlen >= 15u ? 1u + (mlen - 15u) / 255u : 0u);
			const uint32_t tot = live ? lb + mb : 0u;
			uint32_t inc = tot;
#pragma unroll
			for (int d = 1; d < 32; d <<= 1) {
				const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
				if (lane >= d) inc += t;
			}
			const uint32_t opk = op + inc - tot;
			if (live) {
				if (e > matchlimit) bad = true;
				else if (e < matchlimit && src[e] == src[e - o]) bad = true;            // not extended to the end
				if (litlen > 0u && m > o && src[m - 1u] == src[m - o - 1u]) bad = true;  // walk-back stops too early
				if (opk + 1u + litlen + (2u + 1u + LZ4_LASTLITERALS) + (litlen >> 8) > osize) bad = true;
				if (opk + lb + 2u + (1u + LZ4_LASTLITERALS) + (mlen >> 8) > osize) bad = true;
			}
			op += __shfl_sync(0xffffffffu, inc, 31);
			const uint32_t lastlive = (ns - k0 < 32u) ? (ns - k0 - 1u) : 31u;
			prev_e = __shfl_sync(0xffffffffu, e, (int)lastlive);
		}
		const uint32_t last = iend - prev_e;
		if (op + last + 1u + ((last + 255u - 15u) / 255u) > osize) bad = true;
		if (op + 1u + (last >= 15u ? 1u + (last - 15u) / 255u : 0u) + last != clen) bad = true;
	}
	if (__any_sync(0xffffffffu, bad)) return false;

	// ---- the table trajectory
	TAB tab; tab.t = tabmem;
	tab.clear(lane);
	__syncwarp();
	TabRound<TAB> rd;
	// deferred MISS check of the previous round: the candidate's two source words are REQUESTED when the
	// round ends and only looked at when the next one does (a load's first consumer stalls the warp:
	// nothing here may touch the words early, not even the funnel shift that aligns them)
	uint32_t p_lo = 0, p_hi = 0, p_sh = 0, p_v = 1;
#define CHK_EVAL() { bad = bad || (__funnelshift_r(p_lo, p_hi, p_sh) == p_v); }
#define CHK_ISSUE(chk_, pred_, v_)                                                                   \
	{                                                                                                \
		const uint32_t cx_ = (pred_) + mis;                                                          \
		p_lo = (chk_) ? __ldg(base4 + (cx_ >> 2)) : 0u;                                              \
		p_hi = (chk_) ? __ldg(base4 + (cx_ >> 2) + 1u) : 0u;                                         \
		p_sh = (cx_ & 3u) * 8u;                                                                      \
		p_v = (chk_) ? (v_) : 1u;                                                                    \
	}
	uint32_t a = 0;                        // anchor: end of the previous match
	bool follow_hit = false;               // the probe at `a` delivered sequence k (no search)
	uint32_t k = 0;
	// Nothing the chain waits for comes from global memory: lane L keeps sequence kw+L of the parse
	// (w_s) with the two source words its post pair will hash (w_vm2 at e-2, w_ve at e), refilled 16
	// sequences ahead of use, and the first round of the next search is requested one step early
	// from where this step's hypothesis says it will start (pf_start / pf_v).
	uint32_t kw = 0;
	uint64_t w_s = 0; uint32_t w_0 = 0, w_1 = 0, w_2 = 0;   // the three aligned words that hold [e-2, e+4)
	uint32_t pf_start = 0xffffffffu, pf_lo = 0, pf_hi = 0;
	bool w_init = false;
	for (;;) {
		if (__any_sync(0xffffffffu, bad)) return false;      // (a foreign encoder's block usually fails early)
		const bool have = k < ns;
		if (have && (!w_init || k - kw > 15u)) {
			kw = k; w_init = true;
			const uint32_t j = kw + (uint32_t)lane;
			w_s = (j < ns) ? seqs[j] : 0ull;
			const uint32_t we = SEQ_M(w_s) + SEQ_L(w_s);
			const bool wok = (j < ns) && we <= mflimit && we >= 2u;
			const uint32_t wi = (we - 2u + mis) >> 2;
			w_0 = wok ? __ldg(base4 + wi) : 0u;
			w_1 = wok ? __ldg(base4 + wi + 1u) : 0u;
			w_2 = wok ? __ldg(base4 + wi + 2u) : 0u;
		}
		const uint64_t s = have ? __shfl_sync(0xffffffffu, w_s, (int)(k - kw)) : 0ull;
		const uint32_t m = SEQ_M(s), o = SEQ_O(s), e = m + SEQ_L(s);
		// After a match ending at e the encoder inserts e-2 and probes e; when the probe hits, the
		// next sequence follows on at once and does the same.  A whole run of such "post" pairs is
		// replayed in ONE round (pair t on lanes L0+2t, L0+2t+1) under the hypothesis that the
		// parse tells the truth about which probes hit; the first probe that disagrees ends the run.
		// CHAIN_SETUP: this lane's operation in the run that starts with sequence k on lane L0.
		uint32_t c_xx = 0, c_e = 0, c_onext = 0, c_v = 0;
		bool c_part = false, c_query = false, c_nf = false;
		int c_T = 0;
#define CHAIN_SETUP(L0)                                                                              \
		{                                                                                            \
			const int rl_ = lane - (L0);                                                             \
			const bool in_ = rl_ >= 0;                                                               \
			const uint32_t t_ = in_ ? (uint32_t)rl_ >> 1 : 0u;                                       \
			const uint32_t kk_ = k + t_;                                                             \
			const uint32_t ix_ = kk_ - kw;                  /* window lane of the pair's sequence */ \
			const bool ex_ = in_ && kk_ < ns && ix_ <= 30u;                                          \
			const int sl_ = ex_ ? (int)ix_ : 0;                                                      \
			const uint64_t s0_ = __shfl_sync(0xffffffffu, w_s, sl_);                                 \
			const uint64_t sp_ = __shfl_sync(0xffffffffu, w_s, sl_ > 0 ? sl_ - 1 : 0);               \
			const uint64_t sn_ = __shfl_sync(0xffffffffu, w_s, sl_ + 1);                             \
			const uint32_t g0_ = __shfl_sync(0xffffffffu, w_0, sl_);                                 \
			const uint32_t g1_ = __shfl_sync(0xffffffffu, w_1, sl_);                                 \
			const uint32_t g2_ = __shfl_sync(0xffffffffu, w_2, sl_);                                 \
			c_e = SEQ_M(s0_) + SEQ_L(s0_);                                                           \
			const bool fol_ = (t_ == 0u) || (SEQ_M(s0_) == SEQ_M(sp_) + SEQ_L(sp_));                 \
			const bool good_ = ex_ && fol_ && c_e <= mflimit;                                        \
			const uint32_t bm_ = __ballot_sync(0xffffffffu, in_ && (rl_ & 1) && !good_);             \
			c_T = bm_ ? ((__ffs((int)bm_) - 1 - (L0)) >> 1) : ((32 - (L0)) >> 1);                    \
			c_part = in_ && (int)t_ < c_T;                                                           \
			c_query = c_part && (rl_ & 1);                                                           \
			c_xx = (rl_ & 1) ? c_e : c_e - 2u;                                                       \
			{                                                                                        \
				const uint32_t sh_ = ((c_e - 2u + mis) & 3u) * 8u + ((rl_ & 1) ? 16u : 0u);          \
				c_v = (sh_ < 32u) ? __funnelshift_r(g0_, g1_, sh_) : __funnelshift_r(g1_, g2_, sh_ - 32u); \
			}                                                                                        \
			c_nf = (kk_ + 1u < ns) && (SEQ_M(sn_) == c_e);                                           \
			c_onext = SEQ_O(sn_);                                                                    \
			/* the search that follows this run, if the hypothesis holds, starts here */            \
			if (c_T > 0) {                                                                           \
				pf_start = __shfl_sync(0xffffffffu, c_e, (L0) + 2 * c_T - 1) + 1u;                   \
				const uint32_t px_ = pf_start + (uint32_t)lane;                                      \
				const bool pk_ = (px_ + 4u <= iend);                                                 \
				pf_lo = pk_ ? __ldg(base4 + ((px_ + mis) >> 2)) : 0u;                                \
				pf_hi = pk_ ? __ldg(base4 + ((px_ + mis) >> 2) + 1u) : 0u;                           \
			}                                                                                        \
		}
		// CHAIN_FINISH: with `pred` of the round: how many pairs stand, where the encoder is after them
		int c_upto = 0, c_used = 0;
		bool c_hitl = false;
#define CHAIN_FINISH(L0, pred)                                                                       \
		{                                                                                            \
			c_hitl = c_query && c_nf && ((pred) + c_onext == c_xx);                                  \
			const uint32_t mis_ = __ballot_sync(0xffffffffu, c_query && c_nf && !c_hitl);            \
			const int last_ = (L0) + 2 * c_T - 1;                                                    \
			c_upto = mis_ ? (__ffs((int)mis_) - 1) : last_;                                          \
			c_used = ((c_upto - (L0)) >> 1) + 1;                                                     \
			follow_hit = __shfl_sync(0xffffffffu, (int)c_hitl, c_upto) != 0;                         \
			a = __shfl_sync(0xffffffffu, c_e, c_upto);                                               \
		}

		bool post_done = false;
		if (!(have && follow_hit)) {
			const uint32_t start = a + 1u;
			const uint32_t pf_start_in = pf_start, pf_lo_in = pf_lo, pf_hi_in = pf_hi;   // (CHAIN_SETUP below overwrites them)
			const uint32_t target = have ? (m > start ? m : start) : 0xffffffffu;
			bool found = false, finished = false;
			uint32_t a0 = 0;
			int q1l = 32;
			// phase 1: the attempts up to and including the first one at or beyond m.  A literal run
			// longer than one round asks for the next round's source words before working on this one.
			uint32_t xn = 0, n_lo = 0, n_hi = 0;
			for (;;) {
				const uint32_t att = a0 + (uint32_t)lane;
				const uint32_t x = (a0 == 0u) ? start + (uint32_t)lane : xn;
				const uint32_t c_lo = n_lo, c_hi = n_hi;              // (this round's words, if a0 > 0)
				const uint32_t step = (a0 == 0u) ? 1u : ((67u + att) >> 6);
				const bool valid = (x + step <= mflimit);
				int q1, I;                                     // first candidate lane, first lane past mflimit
				uint32_t xq1;
				if (a0 == 0u) {                                // x = start + lane: no votes needed
					q1 = (target - start < 32u) ? (int)(target - start) : 32;
					I = (start + 1u > mflimit) ? 0 : ((mflimit - start < 32u) ? (int)(mflimit - start) : 32);
					xq1 = start + (uint32_t)q1;
				} else {
					const uint32_t cm = __ballot_sync(0xffffffffu, x >= target);
					q1 = cm ? (__ffs((int)cm) - 1) : 32;
					const uint32_t inval = __ballot_sync(0xffffffffu, !valid);
					I = inval ? (__ffs((int)inval) - 1) : 32;
					xq1 = __shfl_sync(0xffffffffu, x, q1 & 31);
				}
				q1l = q1;
				if (q1 == 32 && I == 32) {                     // another round will follow: ask for its words now
					xn = start + skip_dist(att + 32u);
					const bool nk = (xn + 4u <= iend);
					n_lo = nk ? __ldg(base4 + ((xn + mis) >> 2)) : 0u;
					n_hi = nk ? __ldg(base4 + ((xn + mis) >> 2) + 1u) : 0u;
				}
				if (have && I <= q1 && I < 32) return false;            // the encoder runs dry before the hit
				if (q1 < 32 && xq1 + LZ4_MINMATCH > e) return false;
				// the post run rides in the same round when the hypothesis leaves lanes for it
				bool part = valid && lane <= q1;
				bool query = part;
				uint32_t xx = x;
				bool ride = false;
				if (q1 < 30) {
					CHAIN_SETUP(q1 + 1)
					ride = c_T > 0;
					if (ride && c_part) { part = true; query = c_query; xx = c_xx; }
				}
				uint32_t v = 0;
				if (part) {
					if (lane > q1) v = c_v;                                   // post pair: from the window
					else if (a0 == 0u && start == pf_start_in)                // search: requested a step ago
						v = __funnelshift_r(pf_lo_in, pf_hi_in, ((xx + mis) & 3u) * 8u);
					else if (a0 != 0u) v = __funnelshift_r(c_lo, c_hi, ((xx + mis) & 3u) * 8u);
					else v = LDS32(xx);
				}
				const uint32_t h = part ? ((v * 2654435761u) >> (32 - LOG)) : (0xffffffffu - (uint32_t)lane);
				const uint32_t pred = tab_round_query(tab, rd, part, h, xx, lane);
				const bool hit1 = (lane == q1) && part && (pred + o == xx);
				found = __any_sync(0xffffffffu, hit1);
				int upto = (q1 < 32) ? q1 : 31;
				bool ridehit = false;
				if (found && ride) {
					CHAIN_FINISH(q1 + 1, pred)
					upto = c_upto; ridehit = c_hitl;
					k += (uint32_t)c_used;
					post_done = true;
				}
				tab_round_commit(tab, rd, part, h, xx, upto, lane);
				// deferred MISS checks: every committed query that is not a hypothesised-and-delivered hit
				CHK_EVAL()
				const bool chk = part && query && lane <= upto && !hit1 && !ridehit &&
				    (!DIST || pred + LZ4_MAXDIST >= xx);
				CHK_ISSUE(chk, pred, v)
				if (q1 < 32) break;
				if (I < 32) { finished = true; break; }                    // closing search ran dry (have == false here)
				a0 += 32u;
			}
			if (finished) break;
			if (!found) {
				// phase 2: the table did not deliver at the first candidate; keep attempting inside the match
				uint32_t ac = a0 + (uint32_t)q1l + 1u;                   // the attempt after the first candidate
				for (;;) {
					const uint32_t att = ac + (uint32_t)lane;
					const uint32_t x = start + skip_dist(att);
					const uint32_t step = (67u + att) >> 6;
					const bool part = (x + step <= mflimit) && (x + LZ4_MINMATCH <= e);
					if (!__any_sync(0xffffffffu, part)) return false;      // no attempt left that could be the hit
					const uint32_t v = part ? LDS32(x) : 0u;
					const uint32_t h = part ? ((v * 2654435761u) >> (32 - LOG)) : (0xffffffffu - (uint32_t)lane);
					const uint32_t pred = tab_round_query(tab, rd, part, h, x, lane);
					const bool hit = part && (pred + o == x);
					const uint32_t hits = __ballot_sync(0xffffffffu, hit);
					const int F = hits ? (__ffs((int)hits) - 1) : 32;
					tab_round_commit(tab, rd, part, h, x, F < 32 ? F : 31, lane);
					CHK_EVAL()
					const bool chk = part && lane < F && (!DIST || pred + LZ4_MAXDIST >= x);
					CHK_ISSUE(chk, pred, v)
					if (F < 32) break;
					if (!__all_sync(0xffffffffu, part)) return false;
					ac += 32u;
				}
			}
		}
		if (!have) break;
		if (post_done) continue;                                        // (k, a, follow_hit already advanced)
		if (e > mflimit) {
			// the match ends beyond mflimit: the encoder emits its last literals, so this is the last match
			if (k + 1u != ns) return false;
			break;
		}
		{
			CHAIN_SETUP(0)
			const uint32_t v = c_part ? c_v : 0u;
			const uint32_t h = c_part ? ((v * 2654435761u) >> (32 - LOG)) : (0xffffffffu - (uint32_t)lane);
			const uint32_t pred = tab_round_query(tab, rd, c_part, h, c_xx, lane);
			CHAIN_FINISH(0, pred)
			tab_round_commit(tab, rd, c_part, h, c_xx, c_upto, lane);
			k += (uint32_t)c_used;
			CHK_EVAL()
			const bool chk = c_query && lane <= c_upto && !c_hitl && (!DIST || pred + LZ4_MAXDIST >= c_xx);
			CHK_ISSUE(chk, pred, v)
		}
	}
#undef CHAIN_SETUP
#undef CHAIN_FINISH
	CHK_EVAL()
#undef CHK_EVAL
#undef CHK_ISSUE
#undef LDS32
#undef SEQ_M
#undef SEQ_O
#undef SEQ_L
	return !__any_sync(0xffffffffu, bad);
}

// per-warp shared memory: the hash table.  CTA shape: K3_THREADS/32 encoder warps; the launch
// picks as many CTAs per SM as tables fit (24 tables of 8.5 KiB at 4 warps x 6 CTAs, 26 at
// 13 warps x 2 CTAs -- the carve-out has room for 26).
#ifndef K3_THREADS
#define K3_THREADS 128
#endif
#ifndef K3_MIN_BLOCKS
#define K3_MIN_BLOCKS 6
#endif
#define K3_WARPS (K3_THREADS / 32)
template <bool COMPACT>
__global__ void __launch_bounds__(K3_THREADS, K3_MIN_BLOCKS)
k3_lz4_encode(const uint8_t *__restrict__ src_base, uint8_t *__restrict__ dst_base,
    mtz_job *__restrict__ jobs, uint32_t njobs, const uint32_t *__restrict__ skip = nullptr)
{
	extern __shared__ uint4 s_dyn[];
	constexpr uint32_t TABW = COMPACT ? LZ4_TAB_COMPACT_WORDS : LZ4_TAB_BIG_WORDS;
	constexpr uint32_t PERW = TABW;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint32_t *tab = reinterpret_cast<uint32_t *>(s_dyn) + warp * PERW;
	const uint32_t gw = blockIdx.x * K3_WARPS + (uint32_t)warp;
	const uint32_t nw = gridDim.x * K3_WARPS;
	for (uint32_t j = gw; j < njobs; j += nw) {
		if (skip != nullptr && skip[j] != 0u) continue;     // certified: the input frame is the output
		const mtz_job job = jobs[j];
		if (job.lsize == 0u) continue;
		// a compact launch is only made when the host saw nothing but 128 KiB-class
		// blocks; anything else it might meet is stored raw (never wrong, only bigger)
		uint32_t ps;
		if (COMPACT && (job.lsize < (uint32_t)LZ4_64KLIMIT || job.lsize > 131072u))
			ps = job.lsize;
		else
			ps = warp_zfs_lz4_compress<COMPACT>(src_base + job.src_off, job.lsize,
			    dst_base + job.dst_off, tab, lane);
		__syncwarp();
		if (lane == 0) { jobs[j].out_len = ps; jobs[j].status = MTZ_OK; }
	}
}

// K3c: one warp per record.  cert[j] = bytes of the input payload that ARE the output frame
// (4 + clen; the assembler zero-pads to enc[j].out_len), or 0 = not certified (K3 encodes it).
template <bool COMPACT>
__global__ void __launch_bounds__(K3_THREADS, K3_MIN_BLOCKS)
k3c_lz4_certify(const mtz_job *__restrict__ dec, mtz_job *__restrict__ enc,
    const uint32_t *__restrict__ seq_n, uint32_t *__restrict__ cert, uint32_t njobs)
{
	extern __shared__ uint4 s_dyn[];
	constexpr uint32_t TABW = COMPACT ? LZ4_TAB_COMPACT_WORDS : LZ4_TAB_BIG_WORDS;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint32_t *tab = reinterpret_cast<uint32_t *>(s_dyn) + warp * TABW;
	const uint32_t gw = blockIdx.x * K3_WARPS + (uint32_t)warp;
	const uint32_t nw = gridDim.x * K3_WARPS;
	for (uint32_t j = gw; j < njobs; j += nw) {
		const mtz_job jd = dec[j];
		const mtz_job je = enc[j];
		const uint32_t ns = seq_n[j];
		const uint32_t lsize = je.lsize;
		uint32_t c_len = 0, psize = 0;
		bool ok = (jd.lsize != 0u && jd.lsize == lsize && jd.status == MTZ_OK && ns != LZ4_SEQ_NONE);
		// the ranges in which warp_zfs_lz4_compress compresses at all, and this launch's table
		const uint32_t d_len = lsize - (lsize >> 3);
		if (lsize < 1024u || lsize >= (1u << 24) || d_len < 4u) ok = false;
		if (COMPACT && (lsize < (uint32_t)LZ4_64KLIMIT || lsize > 131072u)) ok = false;
		if (ok) {
			const uint8_t *f = reinterpret_cast<const uint8_t *>((uintptr_t)jd.src_off);
			const uint32_t clen = (ld_u8(f) << 24) | (ld_u8(f + 1) << 16) | (ld_u8(f + 2) << 8) | ld_u8(f + 3);
			c_len = clen + 4u;
			psize = (c_len + 511u) & ~511u;
			if (c_len > d_len || psize >= lsize) ok = false;           // zio_compress_data stores it raw
			if (ok) {
				const uint8_t *src = reinterpret_cast<const uint8_t *>((uintptr_t)je.src_off);
				const uint64_t *seqs = reinterpret_cast<const uint64_t *>((uintptr_t)je.dst_off);
				if (COMPACT)
					ok = warp_lz4_certify<Tab17, true>(src, lsize, seqs, ns, clen, d_len - 4u, tab, lane);
				else if (lsize < (uint32_t)LZ4_64KLIMIT)
					ok = warp_lz4_certify<TabU16, false>(src, lsize, seqs, ns, clen, d_len - 4u, tab, lane);
				else
					ok = warp_lz4_certify<TabU32, true>(src, lsize, seqs, ns, clen, d_len - 4u, tab, lane);
			}
		}
		__syncwarp();
		if (lane == 0) {
			cert[j] = ok ? c_len : 0u;
			if (ok) { enc[j].out_len = psize; enc[j].status = MTZ_OK; }
		}
	}
}

} // namespace mtz
