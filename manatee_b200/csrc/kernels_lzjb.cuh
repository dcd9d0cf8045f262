// kernels_lzjb.cuh -- the lzjb and zle frames of the block check in VERIFY (MTZ_FLAG_BLOCK_LZJB).  A
// block ZFS stored with compression=lzjb (3) or zle (14) has a key over that frame, zero-padded to
// PSIZE; k_frame_plan (kernels_frames.cuh) gives each raw record with such a key a job marked with
// its codec (mtz_job.src_len, unused by encode jobs), and these kernels write the frame into the
// record's slot with the declared encoders, restated from ZFS ([EXTERNAL] lzjb.c, zle.c, driven as
// zio_compress_data drives them):
//   d_len = s_len - s_len/8; a result above d_len (the encoders give up with s_len) = stored raw;
//   otherwise the frame is zero-padded to a whole 512-byte sector, and a pad reaching s_len = raw.
// So out_len is the PSIZE of the frame, or lsize = stored raw, the rule k_frame_sums and the checks
// already apply to K3's frames.  A frame never exceeds d_len < lsize: the slots stay disjoint.
//   k_lzjb_encode  one warp per job, the 1024 x u16 lempel table in shared memory (2 KiB per warp)
//   k_zle_encode   one warp per job, zero and literal runs found by ballot
// COMPRESS with MTZ_FLAG_COMPRESSED_IN decodes the lzjb and zle records of a `zfs send -c` stream
// before K3 sees them, with the decoders restated from the same files:
//   k_lzjb_decode  one warp per job, 32 items per round, the output window in shared memory (4 KiB per warp)
//   k_zle_decode   one warp per job, a walk of the length tokens with warp-wide copies and zero fills
// Both keep K2's access contract (include/manatee_gpu.h): read only [src, src+src_len), write only
// [dst, dst+lsize).  ZFS's lzjb loop does not bound its source; these do, and a frame whose decode
// would read at or past the end of its payload is MTZ_ECODEC like a frame ZFS rejects.
#pragma once
#include "kernels_block.cuh"

namespace mtz {

#define LZJB_THREADS 256
#define LZJB_WARPS (LZJB_THREADS / 32)
#define LZJB_MATCH_MIN 3u
#define LZJB_MATCH_MAX 66u          // (1 << MATCH_BITS) + MATCH_MIN - 1, MATCH_BITS 6
#define LZJB_OFFSET_MASK 1023u
#define LZJB_LEMPEL 1024u
#define ZLE_N 64u

// zio_compress_data's rule for a compressor result c_len of an s_len block whose frame is at dst
__device__ __forceinline__ uint32_t zio_sector_pad(uint8_t *dst, uint32_t c_len, uint32_t s_len, int lane)
{
	const uint32_t d_len = s_len - (s_len >> 3);
	if (c_len > d_len) return s_len;
	const uint32_t ps = (c_len + 511u) & ~511u;
	if (ps >= s_len) return s_len;
	for (uint32_t i = c_len + (uint32_t)lane; i < ps; i += 32u) dst[i] = 0;
	return ps;
}

// lzjb_compress(src, dst, s_len, d_len) of a buffer at address phase 0 (1 KiB aligned, as ZFS's
// page-aligned buffers of 128 KiB-class blocks are).  The C table holds the low 16 bits of source
// pointers and takes the offset as (addr(src) - entry) & 1023: for a written slot that is the
// distance, for a never-written one (0) addr(src) & 1023, i.e. the position at phase 0.  So an
// entry here is (uint16_t)position, 0 for "never written", and the offset (pos - entry) & 1023.
//
// Speculative rounds of 32 positions, K3's technique (DESIGN §4): every lane takes its position as
// if all earlier ones in the round were literals, hashes it and reads its slot, forwarding from the
// latest earlier lane of the round with the same slot.  The first lane whose candidate matches is
// the round's last item: the lanes up to it commit their table writes (the latest lane of each slot
// writes), the later lanes are discarded.  Items before the match are literals, so each item's
// output position is closed-form: one copymap byte before each 8th item, 1 byte per literal.  The
// give-up test runs at each copymap byte, where the C code runs it.  Returns the frame length, or
// s_len when the encoder gives up.
__device__ __forceinline__ uint32_t warp_lzjb_compress(const uint8_t *__restrict__ src, uint32_t s_len,
    uint8_t *__restrict__ dst, uint16_t *tab, int lane)
{
	const uint32_t FULL = 0xffffffffu;
	const int32_t d_len = (int32_t)(s_len - (s_len >> 3));
	__syncwarp();
	for (uint32_t i = (uint32_t)lane; i < LZJB_LEMPEL / 2u; i += 32u) reinterpret_cast<uint32_t *>(tab)[i] = 0u;
	__syncwarp();
	const int64_t last_hashed = (int64_t)s_len - (int64_t)LZJB_MATCH_MAX;  // later positions are literals
	uint32_t p = 0, dpos = 0, items = 0, cm_pos = 0, cmv = 0;
	const uint32_t below = (1u << lane) - 1u, upto_me = (2u << lane) - 1u;
	while (p < s_len) {
		const uint32_t q = p + (uint32_t)lane;
		const bool valid = q < s_len;
		const bool hashed = valid && (int64_t)q <= last_hashed;
		uint32_t b0 = 0, b1 = 0, b2 = 0, slot = LZJB_LEMPEL + (uint32_t)lane;
		if (valid) b0 = src[q];
		if (hashed) {
			b1 = src[q + 1]; b2 = src[q + 2];
			uint32_t hv = (b0 << 16) | (b1 << 8) | b2;
			hv += hv >> 9;
			hv += hv >> 5;
			slot = hv & (LZJB_LEMPEL - 1u);
		}
		const uint32_t peers = __match_any_sync(FULL, slot);
		const uint32_t earlier = peers & below;
		uint32_t off = 0;
		bool m = false;
		if (hashed) {
			const uint32_t e = earlier ? p + (31u - (uint32_t)__clz(earlier)) : (uint32_t)tab[slot];
			off = (q - e) & LZJB_OFFSET_MASK;
			if (off != 0u && off <= q) {
				const uint8_t *c = src + (q - off);
				m = c[0] == b0 && c[1] == b1 && c[2] == b2;
			}
		}
		const uint32_t mb = __ballot_sync(FULL, m);
		const uint32_t vb = __ballot_sync(FULL, valid);
		const uint32_t k = mb ? (uint32_t)__ffs(mb) - 1u : 31u - (uint32_t)__clz(vb);
		const uint32_t upto_k = (2u << k) - 1u;
		const bool item = (uint32_t)lane <= k;
		// the items' bytes: copymaps in front of items items+i with (items+i) % 8 == 0
		const uint32_t gi = items + (uint32_t)lane;
		const bool iscm = item && (gi & 7u) == 0u;
		const uint32_t ncm = item ? (gi >> 3) - ((items + 7u) >> 3) + 1u : 0u;
		const uint32_t opos = dpos + (uint32_t)lane + ncm;
		if (__any_sync(FULL, iscm && (int32_t)(opos - 1u) >= d_len - 1 - 16)) return s_len;
		// the match, lane-parallel: bytes 3..65 of the source against the candidate
		uint32_t mlen = 1u, moff = 0u;
		if (mb) {
			moff = __shfl_sync(FULL, off, (int)k);
			const uint8_t *s1 = src + p + k, *c1 = s1 - moff;
			const uint32_t i0 = 3u + (uint32_t)lane, i1 = 35u + (uint32_t)lane;
			const uint32_t x0 = __ballot_sync(FULL, s1[i0] != c1[i0]);
			const uint32_t x1 = __ballot_sync(FULL, i1 < LZJB_MATCH_MAX && s1[i1] != c1[i1]);
			mlen = x0 ? 2u + (uint32_t)__ffs(x0) : (x1 ? 34u + (uint32_t)__ffs(x1) : LZJB_MATCH_MAX);
		}
		__syncwarp();                                   // every read of the table is done
		if (hashed && item && (peers & upto_k & ~upto_me) == 0u) tab[slot] = (uint16_t)q;
		// copymap bytes: the round's last one holds the match bit, if any; a match whose group began
		// in an earlier round sets its bit in that group's byte
		const uint32_t cmb = __ballot_sync(FULL, iscm);
		const uint32_t lc = cmb ? 31u - (uint32_t)__clz(cmb) : 32u;
		if (cmb) { cm_pos = __shfl_sync(FULL, opos - 1u, (int)lc); cmv = 0u; }
		if (mb) cmv |= 1u << ((items + k) & 7u);
		if (iscm) dst[opos - 1u] = (uint8_t)((uint32_t)lane == lc ? cmv : 0u);
		if (!cmb && mb && (uint32_t)lane == k) dst[cm_pos] = (uint8_t)cmv;
		if (item) {
			if (mb && (uint32_t)lane == k) {
				dst[opos] = (uint8_t)(((mlen - LZJB_MATCH_MIN) << 2) | (moff >> 8));
				dst[opos + 1u] = (uint8_t)moff;
			} else {
				dst[opos] = (uint8_t)b0;
			}
		}
		const uint32_t ncm_k = __shfl_sync(FULL, ncm, (int)k);
		dpos += k + 1u + ncm_k + (mb ? 1u : 0u);
		items += k + 1u;
		p += k + mlen;
		__syncwarp();
	}
	return dpos;
}

// zle_compress(src, dst, s_len, d_len, 64): a zero run of up to 256 - 64 bytes is one length byte
// (run - 1 + 64); otherwise a literal run of up to 64 bytes that stops before a pair of zero bytes,
// a length byte (count - 1) and the bytes.  The encoder gives up when fewer than 64 bytes are left
// in front of a literal run, and the result counts only when the whole source was consumed.
// Every decision is warp-uniform; the runs are found by ballot over 32 bytes at a time.
__device__ __forceinline__ uint32_t warp_zle_compress(const uint8_t *__restrict__ src, uint32_t s_len,
    uint8_t *__restrict__ dst, int lane)
{
	const uint32_t FULL = 0xffffffffu;
	const int32_t d_len = (int32_t)(s_len - (s_len >> 3));
	uint32_t sp = 0, dp = 0;
	while (sp < s_len && (int32_t)dp < d_len - 1) {
		const uint32_t first = sp, lenpos = dp++;
		if (src[sp] == 0) {
			const uint32_t lim = min(sp + (256u - ZLE_N), s_len);
			uint32_t e = lim;
			for (uint32_t c = sp; c < lim; c += 32u) {
				const uint32_t q = c + (uint32_t)lane;
				const uint32_t nz = __ballot_sync(FULL, q < lim && src[q] != 0);
				if (nz) { e = c + (uint32_t)__ffs(nz) - 1u; break; }
			}
			if (lane == 0) dst[lenpos] = (uint8_t)(e - first - 1u + ZLE_N);
			sp = e;
		} else {
			if (d_len - (int32_t)dp < (int32_t)ZLE_N) break;
			const uint32_t lim = min(sp + ZLE_N, s_len);
			uint32_t e = lim - 1u;                      // the first pair of zeros, or the run's last byte
			for (uint32_t c = sp; c < lim - 1u; c += 32u) {
				const uint32_t q = c + (uint32_t)lane;
				const uint32_t z2 = __ballot_sync(FULL, q < lim - 1u && src[q] == 0 && src[q + 1u] == 0);
				if (z2) { e = c + (uint32_t)__ffs(z2) - 1u; break; }
			}
			if (src[e] != 0) e++;
			for (uint32_t i = (uint32_t)lane; i < e - sp; i += 32u) dst[dp + i] = src[sp + i];
			if (lane == 0) dst[lenpos] = (uint8_t)(e - first - 1u);
			dp += e - sp;
			sp = e;
		}
	}
	return sp == s_len ? dp : s_len;
}

// One warp per job (grid-stride) of the codec BLK_DC_LZJB: the frame into the job's slot, out_len
// by zio_compress_data's rule.  Jobs of other codecs are left alone.
__global__ void __launch_bounds__(LZJB_THREADS)
k_lzjb_encode(mtz_job *__restrict__ jobs, uint32_t njobs)
{
	__shared__ uint32_t s_tab[LZJB_WARPS][LZJB_LEMPEL / 2u];     // 1024 u16 per warp, word-aligned
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t gw = blockIdx.x * LZJB_WARPS + (uint32_t)warp;
	const uint32_t nw = gridDim.x * LZJB_WARPS;
	for (uint32_t j = gw; j < njobs; j += nw) {
		const mtz_job job = jobs[j];
		if (job.lsize == 0u || job.src_len != BLK_DC_LZJB) continue;
		const uint8_t *src = reinterpret_cast<const uint8_t *>((uintptr_t)job.src_off);
		uint8_t *dst = reinterpret_cast<uint8_t *>((uintptr_t)job.dst_off);
		const uint32_t c = warp_lzjb_compress(src, job.lsize, dst,
		    reinterpret_cast<uint16_t *>(s_tab[warp]), lane);
		const uint32_t ps = zio_sector_pad(dst, c, job.lsize, lane);
		__syncwarp();
		if (lane == 0) { jobs[j].out_len = ps; jobs[j].status = MTZ_OK; }
	}
}

// Likewise for the codec BLK_DC_ZLE.
__global__ void __launch_bounds__(LZJB_THREADS)
k_zle_encode(mtz_job *__restrict__ jobs, uint32_t njobs)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t gw = blockIdx.x * LZJB_WARPS + (uint32_t)warp;
	const uint32_t nw = gridDim.x * LZJB_WARPS;
	for (uint32_t j = gw; j < njobs; j += nw) {
		const mtz_job job = jobs[j];
		if (job.lsize == 0u || job.src_len != BLK_DC_ZLE) continue;
		const uint8_t *src = reinterpret_cast<const uint8_t *>((uintptr_t)job.src_off);
		uint8_t *dst = reinterpret_cast<uint8_t *>((uintptr_t)job.dst_off);
		const uint32_t c = warp_zle_compress(src, job.lsize, dst, lane);
		const uint32_t ps = zio_sector_pad(dst, c, job.lsize, lane);
		__syncwarp();
		if (lane == 0) { jobs[j].out_len = ps; jobs[j].status = MTZ_OK; }
	}
}

// ---- decoders -----------------------------------------------------------------------------------
#define LZJB_RING 4096u             // output window per warp: 1023 bytes of history + a round's <= 32 x 66

// lzjb_decompress(src, dst, s_len, lsize): a copymap byte, then 8 items, 1 byte per literal and 2 per
// match (bit set: length (b0 >> 2) + 3, offset ((b0 << 8) | b1) & 1023).  A copymap byte fixes where
// its 8 items start, so a round takes 4 copymap bytes and 32 items, one per lane, from a 96-byte source
// window held in registers (a round reads at most 4 + 64 bytes).  One shuffle scan of the item lengths
// places every output; literals are stored in parallel, matches resolved in item order (a match reads
// only output before its own, so a periodic copy covers an offset below the length).  The output is
// built in a shared-memory ring and streamed to dst in whole words behind the decode.
// A needed item past the end of the source, an offset of 0 (ZFS would copy destination bytes it never
// wrote) or one reaching before dst is MTZ_ECODEC; items past lsize are not read, like the C loop's.
__device__ __forceinline__ int32_t warp_lzjb_decode(const uint8_t *__restrict__ src, uint32_t s_len,
    uint8_t *__restrict__ dst, uint32_t lsize, uint8_t *ring, int lane)
{
	const uint32_t FULL = 0xffffffffu, RMASK = LZJB_RING - 1u;
	const bool wide = ((uintptr_t)dst & 3u) == 0u;
	const uint32_t g = (uint32_t)lane >> 3, b = (uint32_t)lane & 7u;
	uint32_t ip = 0, op = 0, fl = 0;        // next copymap byte, bytes decoded, bytes stored to dst
	while (op < lsize) {
		uint32_t win = 0;                   // source byte ip + k sits in lane k & 31, byte k >> 5
#pragma unroll
		for (uint32_t k = 0; k < 3u; k++) {
			const uint32_t q = ip + 32u * k + (uint32_t)lane;
			if (q < s_len) win |= (uint32_t)src[q] << (8u * k);
		}
		auto byte_at = [&](uint32_t r) -> uint32_t {
			return (__shfl_sync(FULL, win, (int)(r & 31u)) >> (8u * (r >> 5))) & 0xffu;
		};
		// the 4 copymap bytes of the round and where they sit (relative to ip)
		const uint32_t q0 = 0u, c0 = byte_at(q0);
		const uint32_t q1 = q0 + 9u + (uint32_t)__popc(c0), c1 = byte_at(q1);
		const uint32_t q2 = q1 + 9u + (uint32_t)__popc(c1), c2 = byte_at(q2);
		const uint32_t q3 = q2 + 9u + (uint32_t)__popc(c2), c3 = byte_at(q3);
		const uint32_t cm = g == 0u ? c0 : g == 1u ? c1 : g == 2u ? c2 : c3;
		const uint32_t qg = g == 0u ? q0 : g == 1u ? q1 : g == 2u ? q2 : q3;
		const bool ism = (cm >> b) & 1u;
		const uint32_t r = qg + 1u + b + (uint32_t)__popc(cm & ((1u << b) - 1u));
		const uint32_t b0 = byte_at(r), b1 = byte_at(r + 1u);
		const uint32_t len = ism ? (b0 >> 2) + LZJB_MATCH_MIN : 1u;
		const uint32_t off = ((b0 << 8) | b1) & LZJB_OFFSET_MASK;
		uint32_t inc = len;
#pragma unroll
		for (int d = 1; d < 32; d <<= 1) {
			const uint32_t up = __shfl_up_sync(FULL, inc, d);
			if (lane >= d) inc += up;
		}
		const uint32_t o = op + inc - len;
		const bool need = o < lsize;
		const bool bad = need && (ip + qg >= s_len || ip + r + (ism ? 2u : 1u) > s_len ||
		    (ism && (off == 0u || off > o)));
		if (__any_sync(FULL, bad)) return MTZ_ECODEC;
		const uint32_t clen = need ? min(len, lsize - o) : 0u;
		if (need && !ism) ring[o & RMASK] = (uint8_t)b0;
		__syncwarp();
		for (uint32_t mm = __ballot_sync(FULL, need && ism); mm != 0u; mm &= mm - 1u) {
			const int k = __ffs(mm) - 1;
			const uint32_t mo = __shfl_sync(FULL, o, k), moff = __shfl_sync(FULL, off, k);
			const uint32_t ml = __shfl_sync(FULL, clen, k);
			for (uint32_t i = (uint32_t)lane; i < ml; i += 32u)
				ring[(mo + i) & RMASK] = ring[(mo - moff + (moff < ml ? i % moff : i)) & RMASK];
			__syncwarp();
		}
		const uint32_t total = __shfl_sync(FULL, inc, 31);
		if (op + total >= lsize) {
			op = lsize;
		} else {
			op += total;
			ip += q3 + 9u + (uint32_t)__popc(c3);
		}
		// everything decoded so far up to a word boundary (all of it at the end) goes to dst
		const uint32_t fe = op == lsize ? lsize : (op & ~3u);
		if (wide) {
			const uint32_t fw = fe & ~3u;
			for (uint32_t w = fl + 4u * (uint32_t)lane; w < fw; w += 128u)
				*reinterpret_cast<uint32_t *>(dst + w) = *reinterpret_cast<const uint32_t *>(ring + (w & RMASK));
			for (uint32_t i = fw + (uint32_t)lane; i < fe; i += 32u) dst[i] = ring[i & RMASK];
			fl = fw;
		} else {
			for (uint32_t i = fl + (uint32_t)lane; i < fe; i += 32u) dst[i] = ring[i & RMASK];
			fl = fe;
		}
		__syncwarp();
	}
	return MTZ_OK;
}

// zle_decompress(src, dst, s_len, lsize, 64): a length byte n - 1; n <= 64 is a literal run of n bytes,
// otherwise a run of n - 64 zeros.  A run past either end, or a source that ends before lsize bytes,
// is MTZ_ECODEC.  Every decision is warp-uniform.
__device__ __forceinline__ int32_t warp_zle_decode(const uint8_t *__restrict__ src, uint32_t s_len,
    uint8_t *__restrict__ dst, uint32_t lsize, int lane)
{
	uint32_t sp = 0, dp = 0;
	while (sp < s_len && dp < lsize) {
		uint32_t n = 1u + src[sp++];
		if (n <= ZLE_N) {
			if (sp + n > s_len || dp + n > lsize) return MTZ_ECODEC;
			for (uint32_t i = (uint32_t)lane; i < n; i += 32u) dst[dp + i] = src[sp + i];
			sp += n;
		} else {
			n -= ZLE_N;
			if (dp + n > lsize) return MTZ_ECODEC;
			for (uint32_t i = (uint32_t)lane; i < n; i += 32u) dst[dp + i] = 0;
		}
		dp += n;
	}
	return dp == lsize ? MTZ_OK : MTZ_ECODEC;
}

// One warp per job (grid-stride) of a record whose drr_compressiontype is lzjb: the frame
// [src_off, src_off + src_len) decoded to the lsize bytes at dst_off, status MTZ_OK or MTZ_ECODEC.
// Jobs of other records, and empty jobs (lsize 0), are left alone.  `recs` indexes like `jobs`.
__global__ void __launch_bounds__(LZJB_THREADS)
k_lzjb_decode(const mtz_rec *__restrict__ recs, mtz_job *__restrict__ jobs, uint32_t njobs)
{
	__shared__ uint32_t s_ring[LZJB_WARPS][LZJB_RING / 4u];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t gw = blockIdx.x * LZJB_WARPS + (uint32_t)warp;
	const uint32_t nw = gridDim.x * LZJB_WARPS;
	for (uint32_t j = gw; j < njobs; j += nw) {
		const mtz_job job = jobs[j];
		if (job.lsize == 0u || recs[j].comp != BLK_DC_LZJB) continue;
		const int32_t st = warp_lzjb_decode(reinterpret_cast<const uint8_t *>((uintptr_t)job.src_off), job.src_len,
		    reinterpret_cast<uint8_t *>((uintptr_t)job.dst_off), job.lsize,
		    reinterpret_cast<uint8_t *>(s_ring[warp]), lane);
		if (lane == 0) { jobs[j].status = st; jobs[j].out_len = st == MTZ_OK ? job.lsize : 0u; }
	}
}

// Likewise for the records whose drr_compressiontype is zle.
__global__ void __launch_bounds__(LZJB_THREADS)
k_zle_decode(const mtz_rec *__restrict__ recs, mtz_job *__restrict__ jobs, uint32_t njobs)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t gw = blockIdx.x * LZJB_WARPS + (uint32_t)warp;
	const uint32_t nw = gridDim.x * LZJB_WARPS;
	for (uint32_t j = gw; j < njobs; j += nw) {
		const mtz_job job = jobs[j];
		if (job.lsize == 0u || recs[j].comp != BLK_DC_ZLE) continue;
		const int32_t st = warp_zle_decode(reinterpret_cast<const uint8_t *>((uintptr_t)job.src_off), job.src_len,
		    reinterpret_cast<uint8_t *>((uintptr_t)job.dst_off), job.lsize, lane);
		if (lane == 0) { jobs[j].status = st; jobs[j].out_len = st == MTZ_OK ? job.lsize : 0u; }
	}
}

} // namespace mtz
