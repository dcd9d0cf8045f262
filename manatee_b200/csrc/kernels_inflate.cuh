// kernels_inflate.cuh -- the gzip records of a `zfs send -c` stream (COMPRESS with MTZ_FLAG_COMPRESSED_IN
// | MTZ_FLAG_GZIP_IN).  ZFS's gzip-1 .. gzip-9 (drr_compressiontype 5..13) store a zlib stream (RFC 1950
// header, RFC 1951 deflate blocks, big-endian Adler-32) zero-padded to PSIZE.  k_inflate decodes it to
// drr_logical_size bytes before K3 sees them, by zlib's acceptance rule made strict on length: the
// stream must reach its end (trailer checked) inside the payload and give exactly lsize bytes; the
// padding after the trailer is ignored.  Everything else is MTZ_ECODEC (DESIGN §1 lists the cases).
// As zlib's default build (no INFLATE_STRICT), the window size in CINFO does not cap distances.
//   k_inflate  one warp per job (grid-stride), the Huffman tables of the current block in shared memory
//              (InflSmem, 3648 bytes per warp, 28.5 KiB per CTA of 8 warps)
// Decode, then place: every lane steps the same bit buffer through the same symbols (table reads are
// shared-memory broadcasts, no shuffles), lane k keeping the round's k-th symbol; a round is up to 32
// symbols.  The round's literals are then stored in parallel and its matches copied in symbol order by
// the whole warp, reading the window from dst (a match reads only output before its own).  Stored
// blocks are warp-wide copies.  Adler-32 is computed warp-parallel over dst at the end.
// Keeps K2's access contract (include/manatee_gpu.h): reads only [src, src+src_len), writes only
// [dst, dst+lsize).  Bits past the payload's end read as zeros and consuming one is MTZ_ECODEC.
#pragma once
#include "kernels_codec.cuh"

namespace mtz {

#define INFL_THREADS 256
#define INFL_WARPS (INFL_THREADS / 32)
#define INFL_LBITS 10               // primary lookup bits of the literal/length code
#define INFL_DBITS 8                // ... of the distance code (and 7 of the code-length code fit in it)

// one warp's tables (3648 bytes): a primary table entry is symbol | length << 9 for a code of at most
// *BITS bits, 0 otherwise (a longer code: canonical slow path; no code at all: MTZ_ECODEC there)
struct InflSmem {
	uint16_t lit[1u << INFL_LBITS];
	uint16_t dist[1u << INFL_DBITS];  // the code-length code's table while the lengths are read
	uint16_t lit_sym[288];            // symbols in canonical order
	uint16_t dist_sym[32];
	uint16_t lit_cnt[16];             // codes per length
	uint16_t dist_cnt[16];
	uint16_t nxt[16], cbase[16];      // build scratch
	uint8_t lens[320];                // code lengths: literal/length then distance
};

__device__ __forceinline__ uint32_t rev16(uint32_t v)
{
	v = ((v & 0x5555u) << 1) | ((v >> 1) & 0x5555u);
	v = ((v & 0x3333u) << 2) | ((v >> 2) & 0x3333u);
	v = ((v & 0x0f0fu) << 4) | ((v >> 4) & 0x0f0fu);
	return ((v & 0x00ffu) << 8) | ((v >> 8) & 0x00ffu);
}

// the bit buffer: `bits` unconsumed bits in `hold`, the next byte to load at `ip`; bytes at or past
// s_len load as zero (and count: consumed() > 8 * s_len means a bit past the payload was used)
struct InflBits {
	const uint8_t *src;
	uint32_t s_len, ip, bits;
	uint64_t hold;
	__device__ __forceinline__ void refill()
	{
		while (bits <= 32u) {
			if (ip + 4u <= s_len && (((uintptr_t)src + ip) & 3u) == 0u) {
				hold |= (uint64_t)*reinterpret_cast<const uint32_t *>(src + ip) << bits;
				ip += 4u; bits += 32u;
			} else {
				hold |= (uint64_t)(ip < s_len ? src[ip] : 0u) << bits;
				ip++; bits += 8u;
			}
		}
	}
	__device__ __forceinline__ uint32_t take(uint32_t n)
	{
		const uint32_t v = (uint32_t)hold & ((1u << n) - 1u);
		hold >>= n; bits -= n;
		return v;
	}
	__device__ __forceinline__ uint64_t consumed() const { return 8ull * ip - bits; }
	__device__ __forceinline__ bool over() const { return consumed() > 8ull * s_len; }
};

// The canonical code of lens[0..n) into tab (PRIM primary bits), cnt and sym.  zlib's inflate_table
// rule: over-subscribed is an error; incomplete is an error unless the longest code has 1 bit and this
// is not the code-length code; no code at all is accepted (decoding from it then fails).
template <int PRIM>
__device__ __forceinline__ bool warp_huff_build(const uint8_t *lens, uint32_t n, uint16_t *tab, uint16_t *cnt,
    uint16_t *sym, uint16_t *nxt, uint16_t *cbase, bool cl_code, int lane)
{
	const uint32_t FULL = 0xffffffffu, lt = (1u << lane) - 1u;
	__syncwarp();
	if (lane < 16) cnt[lane] = 0;
	for (uint32_t i = (uint32_t)lane; i < (1u << PRIM); i += 32u) tab[i] = 0;
	__syncwarp();
	for (uint32_t b = 0; b < n; b += 32u) {
		const uint32_t s = b + (uint32_t)lane, L = s < n ? lens[s] : 0u;
		const uint32_t m = __match_any_sync(FULL, L);
		if (L != 0u && (m & lt) == 0u) cnt[L] += (uint16_t)__popc(m);
		__syncwarp();
	}
	int left = 1;
	uint32_t off = 0, code = 0, maxl = 0;
	bool bad = false;
	for (uint32_t L = 1; L <= 15u; L++) {
		const uint32_t c = cnt[L];
		left = (left << 1) - (int)c;
		bad |= left < 0;
		if ((uint32_t)lane == L) { nxt[L] = (uint16_t)off; cbase[L] = (uint16_t)(code - off); }
		off += c;
		code = (code + c) << 1;
		if (c) maxl = L;
	}
	if (bad || (left > 0 && maxl != 0u && (cl_code || maxl != 1u))) return false;
	__syncwarp();
	for (uint32_t b = 0; b < n; b += 32u) {
		const uint32_t s = b + (uint32_t)lane, L = s < n ? lens[s] : 0u;
		const uint32_t m = __match_any_sync(FULL, L);
		uint32_t idx = 0;
		if (L != 0u) idx = nxt[L] + (uint32_t)__popc(m & lt);
		__syncwarp();
		if (L != 0u) {
			if ((m & lt) == 0u) nxt[L] = (uint16_t)(nxt[L] + __popc(m));
			sym[idx] = (uint16_t)s;
			if (L <= (uint32_t)PRIM) {
				const uint32_t c = (idx + cbase[L]) & 0xffffu;
				const uint32_t rev = rev16(c) >> (16u - L);
				for (uint32_t k = rev; k < (1u << PRIM); k += 1u << L) tab[k] = (uint16_t)(s | (L << 9));
			}
		}
		__syncwarp();
	}
	return true;
}

// one symbol of the code (tab, cnt, sym): -1 when the bits are no code of it (an incomplete code)
template <int PRIM>
__device__ __forceinline__ int huff_decode(InflBits &br, const uint16_t *tab, const uint16_t *cnt, const uint16_t *sym)
{
	const uint32_t e = tab[(uint32_t)br.hold & ((1u << PRIM) - 1u)];
	if (e != 0u) {
		br.take(e >> 9);
		return (int)(e & 511u);
	}
	int code = 0, first = 0, index = 0;               // longer codes: the canonical walk, bit by bit
	uint64_t h = br.hold;
	for (uint32_t L = 1; L <= 15u; L++) {
		code |= (int)(h & 1u);
		h >>= 1;
		const int c = cnt[L];
		if (code - c < first) {
			br.take(L);
			return sym[index + code - first];
		}
		index += c;
		first = (first + c) << 1;
		code <<= 1;
	}
	return -1;
}

// Adler-32 of [p, p+n), warp-parallel; every lane gets it
__device__ __forceinline__ uint32_t warp_adler32(const uint8_t *p0, uint32_t n, int lane)
{
	const uint32_t FULL = 0xffffffffu;
	uint64_t a = 0, b = 0;
	auto add = [&](uint32_t p, uint32_t v) { a += v; b += (uint64_t)(n - p) * v; };
	uint32_t tail = 0;
	if (((uintptr_t)p0 & 15u) == 0u) {
		tail = n & ~15u;
		for (uint32_t p = 16u * (uint32_t)lane; p < tail; p += 512u) {
			const uint4 v = *reinterpret_cast<const uint4 *>(p0 + p);
			const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
			for (int q = 0; q < 16; q++) add(p + (uint32_t)q, (w[q >> 2] >> (8 * (q & 3))) & 0xffu);
		}
	}
	for (uint32_t p = tail + (uint32_t)lane; p < n; p += 32u) add(p, p0[p]);
	uint32_t sa = (uint32_t)(a % 65521u), sb = (uint32_t)(b % 65521u);
#pragma unroll
	for (int d = 16; d > 0; d >>= 1) {
		sa += __shfl_xor_sync(FULL, sa, d);
		sb += __shfl_xor_sync(FULL, sb, d);
		sa %= 65521u; sb %= 65521u;
	}
	sa = (sa + 1u) % 65521u;
	sb = (uint32_t)((sb + (uint64_t)n) % 65521u);
	return (sb << 16) | sa;
}

// zlib's uncompress of [src, src+s_len) to exactly lsize bytes at dst: MTZ_OK or MTZ_ECODEC
__device__ __forceinline__ int32_t warp_inflate(const uint8_t *__restrict__ src, uint32_t s_len,
    uint8_t *__restrict__ dst, uint32_t lsize, InflSmem &S, int lane)
{
	const uint32_t FULL = 0xffffffffu;
	InflBits br;
	br.src = src; br.s_len = s_len; br.ip = 0; br.bits = 0; br.hold = 0;
	br.refill();
	{
		const uint32_t cmf = br.take(8), flg = br.take(8);
		if ((cmf * 256u + flg) % 31u != 0u || (cmf & 15u) != 8u || (cmf >> 4) > 7u || (flg & 0x20u)) return MTZ_ECODEC;
	}
	uint32_t o = 0;                                    // bytes decoded
	bool last = false, fixed = false;
	while (!last) {
		br.refill();
		last = br.take(1) != 0u;
		const uint32_t type = br.take(2);
		if (type == 0u) {                              // stored
			br.take(br.bits & 7u);
			br.refill();
			const uint32_t len = br.take(16), nlen = br.take(16);
			if (len != (~nlen & 0xffffu)) return MTZ_ECODEC;
			const uint32_t pos = br.ip - br.bits / 8u;
			if (br.ip > s_len + br.bits / 8u || len > s_len - pos || len > lsize - o) return MTZ_ECODEC;
			for (uint32_t i = (uint32_t)lane; i < len; i += 32u) dst[o + i] = src[pos + i];
			o += len;
			br.ip = pos + len; br.bits = 0; br.hold = 0;
			__syncwarp();
			continue;
		}
		if (type == 3u) return MTZ_ECODEC;
		if (type == 1u) {
			if (!fixed) {
				for (uint32_t i = (uint32_t)lane; i < 320u; i += 32u)
					S.lens[i] = (uint8_t)(i < 144u ? 8u : i < 256u ? 9u : i < 280u ? 7u : i < 288u ? 8u : 5u);
				if (!warp_huff_build<INFL_LBITS>(S.lens, 288u, S.lit, S.lit_cnt, S.lit_sym, S.nxt, S.cbase, false, lane) ||
				    !warp_huff_build<INFL_DBITS>(S.lens + 288, 32u, S.dist, S.dist_cnt, S.dist_sym, S.nxt, S.cbase, false, lane))
					return MTZ_ECODEC;
				fixed = true;
			}
		} else {
			fixed = false;
			const uint32_t nlit = br.take(5) + 257u;
			const uint32_t ndist = br.take(5) + 1u, nclen = br.take(4) + 4u;
			if (nlit > 286u || ndist > 30u) return MTZ_ECODEC;
			__syncwarp();
			for (uint32_t i = (uint32_t)lane; i < 19u; i += 32u) S.lens[i] = 0;
			__syncwarp();
			for (uint32_t i = 0; i < nclen; i++) {
				br.refill();
				const uint32_t v = br.take(3);
				// RFC 1951 3.2.7: the order of the code-length code's lengths
				const uint32_t at = i == 0u ? 16u : i == 1u ? 17u : i == 2u ? 18u : i == 3u ? 0u :
				    ((i - 4u) & 1u) ? 7u - (i - 4u) / 2u : 8u + (i - 4u) / 2u;
				if (lane == 0) S.lens[at] = (uint8_t)v;
			}
			if (!warp_huff_build<7>(S.lens, 19u, S.dist, S.dist_cnt, S.dist_sym, S.nxt, S.cbase, true, lane))
				return MTZ_ECODEC;
			const uint32_t total = nlit + ndist;
			uint32_t i = 0, prev = 0;
			while (i < total) {
				br.refill();
				const int s = huff_decode<7>(br, S.dist, S.dist_cnt, S.dist_sym);
				if (s < 0) return MTZ_ECODEC;
				if (s < 16) {
					if (lane == 0) S.lens[i] = (uint8_t)s;
					prev = (uint32_t)s;
					i++;
					continue;
				}
				uint32_t rep, v = 0;
				if (s == 16) {
					if (i == 0u) return MTZ_ECODEC;
					v = prev; rep = 3u + br.take(2);
				} else if (s == 17) {
					rep = 3u + br.take(3);
				} else {
					rep = 11u + br.take(7);
				}
				if (rep > total - i) return MTZ_ECODEC;
				for (uint32_t k = (uint32_t)lane; k < rep; k += 32u) S.lens[i + k] = (uint8_t)v;
				prev = v;
				i += rep;
			}
			__syncwarp();
			if (S.lens[256] == 0u) return MTZ_ECODEC;
			if (!warp_huff_build<INFL_LBITS>(S.lens, nlit, S.lit, S.lit_cnt, S.lit_sym, S.nxt, S.cbase, false, lane) ||
			    !warp_huff_build<INFL_DBITS>(S.lens + nlit, ndist, S.dist, S.dist_cnt, S.dist_sym, S.nxt, S.cbase, false, lane))
				return MTZ_ECODEC;
		}
		// the block's symbols, a round of up to 32 at a time
		bool eob = false;
		while (!eob) {
			uint32_t kind = 0, mo = 0, ml = 0, md = 0;    // lane k: the round's k-th symbol (1 literal, 2 match)
			for (uint32_t k = 0; k < 32u; k++) {
				br.refill();
				const int s = huff_decode<INFL_LBITS>(br, S.lit, S.lit_cnt, S.lit_sym);
				if (s < 0) return MTZ_ECODEC;
				if (s < 256) {
					if (o >= lsize) return MTZ_ECODEC;
					if ((uint32_t)lane == k) { kind = 1u; mo = o; ml = (uint32_t)s; }
					o++;
					continue;
				}
				if (s == 256) { eob = true; break; }
				if (s >= 286) return MTZ_ECODEC;
				const uint32_t li = (uint32_t)s - 257u;
				uint32_t len;
				if (li < 8u) len = 3u + li;
				else if (li == 28u) len = 258u;
				else {
					const uint32_t eb = (li - 4u) >> 2;
					len = ((4u + (li & 3u)) << eb) + 3u + br.take(eb);
				}
				br.refill();
				const int ds = huff_decode<INFL_DBITS>(br, S.dist, S.dist_cnt, S.dist_sym);
				if (ds < 0 || ds >= 30) return MTZ_ECODEC;
				uint32_t dist;
				if (ds < 4) dist = (uint32_t)ds + 1u;
				else {
					const uint32_t eb = ((uint32_t)ds >> 1) - 1u;
					dist = ((2u + ((uint32_t)ds & 1u)) << eb) + 1u + br.take(eb);
				}
				if (dist > o || len > lsize - o) return MTZ_ECODEC;
				if ((uint32_t)lane == k) { kind = 2u; mo = o; ml = len; md = dist; }
				o += len;
			}
			if (br.over()) return MTZ_ECODEC;
			// place the round: literals at once, then the matches in symbol order
			if (kind == 1u) dst[mo] = (uint8_t)ml;
			__syncwarp();
			for (uint32_t mm = __ballot_sync(FULL, kind == 2u); mm != 0u; mm &= mm - 1u) {
				const int k = __ffs(mm) - 1;
				const uint32_t at = __shfl_sync(FULL, mo, k), n = __shfl_sync(FULL, ml, k), d = __shfl_sync(FULL, md, k);
				const uint8_t *from = dst + at - d;
				if (d >= n) {
					for (uint32_t i = (uint32_t)lane; i < n; i += 32u) dst[at + i] = from[i];
				} else if (d >= 32u) {                  // each 32 bytes read only bytes already written
					for (uint32_t c = 0; c < n; c += 32u) {
						const uint32_t i = c + (uint32_t)lane;
						if (i < n) dst[at + i] = from[i];
						__syncwarp();
					}
				} else {                                // period d < 32: one load, then shuffles
					uint32_t r = (uint32_t)lane % d;
					const uint32_t p = from[r], step = 32u % d;
					for (uint32_t c = 0; c < n; c += 32u) {
						const uint32_t v = __shfl_sync(FULL, p, (int)r);
						if (c + (uint32_t)lane < n) dst[at + c + (uint32_t)lane] = (uint8_t)v;
						r += step;
						if (r >= d) r -= d;
					}
				}
				__syncwarp();
			}
		}
	}
	// the trailer: Adler-32 of the output, big endian, from the next byte boundary
	br.take(br.bits & 7u);
	br.refill();
	const uint32_t t = br.take(16), t2 = br.take(16);
	const uint32_t want = ((t & 0xffu) << 24) | ((t >> 8) << 16) | ((t2 & 0xffu) << 8) | (t2 >> 8);
	if (br.over() || o != lsize) return MTZ_ECODEC;
	__syncwarp();
	return warp_adler32(dst, lsize, lane) == want ? MTZ_OK : MTZ_ECODEC;
}

// One warp per job (grid-stride) of a record whose drr_compressiontype is gzip-1 .. gzip-9: the zlib
// stream [src_off, src_off + src_len) inflated to the lsize bytes at dst_off, status MTZ_OK or
// MTZ_ECODEC.  Jobs of other records, and empty jobs (lsize 0), are left alone.  `recs` indexes like `jobs`.
__global__ void __launch_bounds__(INFL_THREADS)
k_inflate(const mtz_rec *__restrict__ recs, mtz_job *__restrict__ jobs, uint32_t njobs)
{
	__shared__ InflSmem s_w[INFL_WARPS];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t gw = blockIdx.x * INFL_WARPS + (uint32_t)warp;
	const uint32_t nw = gridDim.x * INFL_WARPS;
	for (uint32_t j = gw; j < njobs; j += nw) {
		const mtz_job job = jobs[j];
		if (job.lsize == 0u || !is_gzip(recs[j].comp)) continue;
		const int32_t st = warp_inflate(reinterpret_cast<const uint8_t *>((uintptr_t)job.src_off), job.src_len,
		    reinterpret_cast<uint8_t *>((uintptr_t)job.dst_off), job.lsize, s_w[warp], lane);
		if (lane == 0) { jobs[j].status = st; jobs[j].out_len = st == MTZ_OK ? job.lsize : 0u; }
	}
}

} // namespace mtz
