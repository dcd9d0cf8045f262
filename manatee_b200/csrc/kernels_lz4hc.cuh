// kernels_lz4hc.cuh -- K3h: the high-ratio LZ4 encoder of MTZ_FLAG_LZ4_HC (COMPRESS), sm_90a.
//
// Same job contract as K3 (k3_lz4_encode), a different parse: a 16-way hash chain with a 64-byte
// capped candidate comparison instead of ZFS's one-candidate skip-ahead search.  The parse is
// specified exactly (DESIGN.md section 1) and restated serially by tests/lz4hc_ref.c, which this
// kernel equals byte for byte:
//   hash(p) = (LE32(src+p) * 2654435761) >> 20, 4096 buckets of the last 16 positions inserted with
//   that hash; every position below p is inserted before p is searched; the candidates at p < n-12
//   are the bucket's entries c with p-c <= 65535 and LE32(c) == LE32(p), each compared for at most
//   min(64, n-5-p) bytes; the longest wins (the larger c on a tie) and only it is extended to n-5.
//
// One warp per record, persistent grid.  Bucket b of a warp is 16 u32 slots in device scratch
// (LZ4HC_TAB_BYTES per warp) plus an insertion count in shared memory.  The counts are zeroed per
// block, and a slot is visible only while its index is below its bucket's count (or the bucket has
// wrapped), so no entry of an earlier block is ever read and the scratch is never cleared.
//   literal runs  32 consecutive positions per round, one per lane; a lane's candidates are its
//                 bucket's newest entries plus the older lanes of the round with the same hash
//                 (__match_any_sync), so every lane sees exactly the serial table.  The first lane
//                 with a candidate is the next match.
//   insertion     32 positions per step; lanes with the same hash rank themselves and only the
//                 newest 16 of a bucket write, which equals serial insertion.
//   extension     the winner alone, cooperatively in 128-byte rounds.
#pragma once
#include "kernels_lz4.cuh"

namespace mtz {

#define LZ4HC_HB      12
#define LZ4HC_BUCKETS (1u << LZ4HC_HB)
#define LZ4HC_W       16u
#define LZ4HC_CAP     64u
#define LZ4HC_TAB_BYTES ((size_t)LZ4HC_BUCKETS * LZ4HC_W * sizeof(uint32_t))    // 256 KiB per warp
#define LZ4HC_THREADS 64
#define LZ4HC_WARPS   (LZ4HC_THREADS / 32)
#define LZ4HC_CTAS_PER_SM 2                     // 4 warps per SM: the table scratch is sized by it

// The block's bytes through aligned 32-bit words: word i of base4 is read only when it starts
// before the 4-byte boundary at or after the block's end (wend).
struct HcSrc {
	const uint32_t *base4;
	uint32_t mis, wend;
	__device__ __forceinline__ uint32_t ld(uint32_t pos) const {
		const uint32_t x = pos + mis, i = x >> 2;
		const uint32_t lo = __ldg(base4 + i);
		const uint32_t hi = (i + 1u < wend) ? __ldg(base4 + i + 1u) : 0u;
		return __funnelshift_r(lo, hi, (x & 3u) * 8u);
	}
};

__device__ __forceinline__ uint32_t hc_hash(uint32_t v) { return (v * 2654435761u) >> (32 - LZ4HC_HB); }

// insert the positions q of the warp's lanes (consecutive, lane order; `grp` = __match_any_sync of h)
__device__ __forceinline__ void hc_insert_step(uint32_t *__restrict__ tab, uint32_t *cnt, uint32_t q, bool valid,
    uint32_t h, uint32_t grp, int lane)
{
	const uint32_t rank = __popc(grp & ((1u << lane) - 1u)), total = __popc(grp);
	uint32_t c = 0;
	if (valid) c = cnt[h];
	__syncwarp();
	if (valid && total - rank <= LZ4HC_W) tab[h * LZ4HC_W + ((c + rank) & (LZ4HC_W - 1u))] = q;
	if (valid && rank == total - 1u) cnt[h] = c + total;
	__syncwarp();
}

// insert positions [lo, hi) in order (warp-uniform arguments)
__device__ __forceinline__ void hc_insert(const HcSrc &s, uint32_t *__restrict__ tab, uint32_t *cnt,
    uint32_t lo, uint32_t hi, int lane)
{
	for (uint32_t b = lo; b < hi; b += 32u) {
		const uint32_t q = b + (uint32_t)lane;
		const bool valid = q < hi;
		const uint32_t h = valid ? hc_hash(s.ld(q)) : (LZ4HC_BUCKETS + (uint32_t)lane);  // invalid: own group
		hc_insert_step(tab, cnt, q, valid, h, __match_any_sync(0xffffffffu, h), lane);
	}
}

// cooperative store of `len` bytes src[from, from+len) at dst[op]
__device__ __forceinline__ void hc_copy(uint8_t *__restrict__ dst, uint32_t op, const uint8_t *__restrict__ src,
    uint32_t from, uint32_t len, int lane)
{
	for (uint32_t i = (uint32_t)lane; i < len; i += 32u) dst[op + i] = src[from + i];
}

// bytes of a sequence with `lit` literals and match length ml (0 = the closing literals-only one)
__device__ __forceinline__ uint32_t hc_seq_bytes(uint32_t lit, uint32_t ml)
{
	uint32_t n = 1u + lit + (lit >= 15u ? (lit - 15u) / 255u + 1u : 0u);
	if (ml) n += 2u + (ml - 4u >= 15u ? (ml - 19u) / 255u + 1u : 0u);
	return n;
}

// one sequence at dst[op] (warp-uniform arguments); returns the new op
__device__ __forceinline__ uint32_t hc_put_seq(uint8_t *__restrict__ dst, uint32_t op, const uint8_t *__restrict__ src,
    uint32_t anchor, uint32_t lit, uint32_t off, uint32_t ml, int lane)
{
	const uint32_t mc = ml ? ml - 4u : 0u;
	if (lane == 0) dst[op] = (uint8_t)(((lit >= 15u ? 15u : lit) << 4) | (mc >= 15u ? 15u : mc));
	op += 1u;
	if (lit >= 15u) op = put_len_ext(dst, op, lit - 15u, lane);
	hc_copy(dst, op, src, anchor, lit, lane);
	op += lit;
	if (ml == 0u) return op;
	if (lane == 0) { dst[op] = (uint8_t)off; dst[op + 1] = (uint8_t)(off >> 8); }
	op += 2u;
	if (mc >= 15u) op = put_len_ext(dst, op, mc - 15u, lane);
	return op;
}

// Raw LZ4 block of src[0, n) into dst[0, osize); returns its length, 0 if it does not fit.
__device__ uint32_t warp_lz4hc_encode(const uint8_t *__restrict__ src, uint32_t n, uint8_t *__restrict__ dst,
    uint32_t osize, uint32_t *__restrict__ tab, uint32_t *cnt, int lane)
{
	HcSrc s;
	s.mis = (uint32_t)((uintptr_t)src & 3u);
	s.base4 = reinterpret_cast<const uint32_t *>(src - s.mis);
	s.wend = (s.mis + n + 3u) >> 2;
	for (uint32_t i = (uint32_t)lane; i < LZ4HC_BUCKETS; i += 32u) cnt[i] = 0;
	__syncwarp();

	const uint32_t lower = (1u << lane) - 1u;
	uint32_t p = 0, anchor = 0, op = 0;
	if (n > (uint32_t)LZ4_MFLIMIT) {
		const uint32_t mflimit = n - LZ4_MFLIMIT, matchlimit = n - LZ4_LASTLITERALS;
		while (p < mflimit) {
			// ---- one round: positions p .. p+31, every position below p already inserted
			const uint32_t q = p + (uint32_t)lane;
			const bool valid = q < mflimit;
			uint32_t v = 0, h = LZ4HC_BUCKETS + (uint32_t)lane;
			if (valid) { v = s.ld(q); h = hc_hash(v); }
			const uint32_t grp = __match_any_sync(0xffffffffu, h);
			uint32_t best = 0, bc = 0;
			if (valid) {
				const uint32_t lim = min(LZ4HC_CAP, matchlimit - q);
				const uint32_t c0 = cnt[h];
				uint32_t fw = grp & lower;                          // older lanes, same bucket
				while (__popc(fw) > (int)LZ4HC_W) fw &= fw - 1u;    // only the newest 16 survive
				const uint32_t nf = __popc(fw);
				const uint32_t nt = min(min(c0, LZ4HC_W), LZ4HC_W - nf);
				for (uint32_t k = 0; k < nt + nf; k++) {
					uint32_t c;
					if (k < nt) {
						c = tab[h * LZ4HC_W + ((c0 - 1u - k) & (LZ4HC_W - 1u))];
					} else {
						c = p + (uint32_t)(31 - __clz((int)fw));
						fw &= ~(1u << (c - p));
					}
					if (q - c > (uint32_t)LZ4_MAXDIST || s.ld(c) != v) continue;
					uint32_t len = 4u;
					for (; len < lim; len += 4u) {
						const uint32_t x = s.ld(c + len) ^ s.ld(q + len);
						if (x) { len += (uint32_t)(__ffs((int)x) - 1) >> 3; break; }
					}
					len = min(len, lim);
					if (len > best || (len == best && c > bc)) { best = len; bc = c; }
				}
			}
			const uint32_t hits = __ballot_sync(0xffffffffu, best != 0u);
			if (hits == 0u) {                                       // the round's positions go in as they are
				hc_insert_step(tab, cnt, q, valid, h, grp, lane);
				p = min(p + 32u, mflimit);
				continue;
			}
			const int F = __ffs((int)hits) - 1;
			const uint32_t m = p + (uint32_t)F;
			const uint32_t c = __shfl_sync(0xffffffffu, bc, F);
			uint32_t ml = __shfl_sync(0xffffffffu, best, F);
			if (ml == LZ4HC_CAP) {
				// ---- extend the winner in 128-byte rounds up to matchlimit
				for (uint32_t e = m + LZ4HC_CAP;; e += 128u) {
					const uint32_t o = e + 4u * (uint32_t)lane;
					const uint32_t room = (o < matchlimit) ? matchlimit - o : 0u;
					uint32_t k = 0;
					if (room) {
						const uint32_t x = s.ld(o) ^ s.ld(o - m + c);
						k = x ? (uint32_t)(__ffs((int)x) - 1) >> 3 : 4u;
						k = min(k, room);
					}
					const uint32_t part = __ballot_sync(0xffffffffu, k < 4u);
					if (part) {
						const int Fp = __ffs((int)part) - 1;
						ml = e + 4u * (uint32_t)Fp + __shfl_sync(0xffffffffu, k, Fp) - m;
						break;
					}
				}
			}
			// ---- emit (literals [anchor, m), offset m-c, ml), then insert [p, m+ml)
			const uint32_t lit = m - anchor;
			if (op + hc_seq_bytes(lit, ml) > osize) return 0u;
			op = hc_put_seq(dst, op, src, anchor, lit, m - c, ml, lane);
			hc_insert(s, tab, cnt, p, min(m + ml, mflimit), lane);
			p = m + ml;
			anchor = p;
		}
	}
	const uint32_t last = n - anchor;
	if (op + hc_seq_bytes(last, 0u) > osize) return 0u;
	op = hc_put_seq(dst, op, src, anchor, last, 0u, 0u, lane);
	__syncwarp();
	return op;
}

// K3h: k3_lz4_encode's contract (frame or store-raw per job: out_len = psize or lsize, status MTZ_OK,
// writes only inside the lsize-byte frame slot) with this parse.  `tabs`: LZ4HC_TAB_BYTES per warp
// of the grid.
__global__ void __launch_bounds__(LZ4HC_THREADS)
k3h_lz4hc_encode(const uint8_t *__restrict__ src_base, uint8_t *__restrict__ dst_base,
    mtz_job *__restrict__ jobs, uint32_t njobs, uint32_t *__restrict__ tabs)
{
	__shared__ uint32_t s_cnt[LZ4HC_WARPS][LZ4HC_BUCKETS];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t gw = blockIdx.x * LZ4HC_WARPS + (uint32_t)warp;
	const uint32_t nw = gridDim.x * LZ4HC_WARPS;
	uint32_t *tab = tabs + (size_t)gw * (LZ4HC_TAB_BYTES / sizeof(uint32_t));
	for (uint32_t j = gw; j < njobs; j += nw) {
		const mtz_job job = jobs[j];
		if (job.lsize == 0u) continue;
		const uint32_t lsize = job.lsize, d_len = lsize - (lsize >> 3);
		uint32_t ps = lsize;
		if (lsize >= 1024u && lsize <= (16u << 20)) {
			uint8_t *dst = dst_base + job.dst_off;
			const uint32_t blk = warp_lz4hc_encode(src_base + job.src_off, lsize, dst + 4, d_len - 4u,
			    tab, s_cnt[warp], lane);
			const uint32_t c_len = blk + 4u;
			if (blk != 0u && c_len <= d_len && ((c_len + 511u) & ~511u) < lsize) {
				ps = (c_len + 511u) & ~511u;
				if (lane == 0) {
					dst[0] = (uint8_t)(blk >> 24); dst[1] = (uint8_t)(blk >> 16);
					dst[2] = (uint8_t)(blk >> 8);  dst[3] = (uint8_t)blk;
				}
				for (uint32_t i = c_len + (uint32_t)lane; i < ps; i += 32u) dst[i] = 0;
			}
		}
		__syncwarp();
		if (lane == 0) { jobs[j].out_len = ps; jobs[j].status = MTZ_OK; }
	}
}

} // namespace mtz
