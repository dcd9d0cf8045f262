// kernels_deflate.cuh -- MTZ_FLAG_GZIP_ENCODE: K3's LZ4 parse of a record re-coded as one dynamic-Huffman
// deflate block in a zlib stream (RFC 1950 / 1951), the frame gzip-1 records carry on the compressed wire.
// The frame is normative: tests/gzip_encode_ref.py states it and this kernel writes it byte for byte.
//   symbols  K3's sequences in order: each literal a literal symbol; a match with offset > 32768 the
//            literal symbols of the bytes it covers (read from the logical input, as all literals are);
//            any other match cut into pieces of at most 258 (match_piece: 259 -> 256 + 3, 260 -> 257 + 3);
//            then end-of-block
//   codes    huffman lengths by warp_huff_lengths (15 bits, 7 for the code-length code); a record without
//            matches sends one distance code of length 1 (zlib's convention)
//   frame    CMF 0x78, FLG 0x01, BFINAL = 1, BTYPE = 2, the block, byte alignment, Adler-32 big endian, zero
//            padding to a multiple of 512 bytes
// k_deflate_from_lz4: one warp per record (grid-stride).  Walk 1 over the LZ4 sequences builds the
// histograms in shared memory; the warp builds the three codes; from them the exact frame size is known,
// and only a frame that is used is written.  Walk 2 gathers up to 32 items (a literal, or the length or
// the distance half of a match piece) a round, places them by a warp prefix sum of their bit widths
// into a shared word buffer and stores every completed 32-bit word.  No symbol buffer is kept.
#pragma once
#include "kernels_inflate.cuh"

namespace mtz {

#define DEFL_THREADS 128
#define DEFL_WARPS (DEFL_THREADS / 32)
#define DEFL_MAXDIST 32768u
#define DEFL_BUFW 36u                       // word buffer: one round is at most 32 x 32 bits + a carried word

// one warp's shared memory (7.4 KiB)
struct DeflSmem {
	uint32_t lf[288];                   // literal/length frequencies, then code | length << 16
	uint32_t df[32];                    // distance frequencies, then likewise
	uint32_t cf[20];                    // code-length code frequencies, then likewise
	uint32_t w[288];                    // huffman build: working frequencies
	uint32_t iw[288];                   // ... weights of the internal nodes
	uint16_t ord[288];                  // ... used symbols sorted by (frequency, symbol)
	uint16_t lpar[288], ipar[288];      // ... parent (internal node) of each sorted leaf / internal node
	uint8_t idep[288];                  // ... depth of each internal node
	uint8_t len[320];                   // code lengths: literal/length 0..287, distance 288..319
	uint8_t clen[20];                   // code-length code lengths
	uint16_t cls[320];                  // the code-length symbols: symbol | extra << 5
	uint32_t buf[DEFL_BUFW];
	uint32_t cnt[16], nxt[16];
};

__device__ __forceinline__ uint32_t defl_lcode(uint32_t L)          // match length 3..258 -> 0..28
{
	if (L < 11u) return L - 3u;
	if (L == 258u) return 28u;
	const uint32_t v = L - 3u, e = 29u - __clz(v);                  // floor(log2 v) - 2
	return 4u * e + 4u + ((v >> e) & 3u);
}
__device__ __forceinline__ uint32_t defl_lextra(uint32_t c) { return c < 8u || c == 28u ? 0u : (c - 4u) >> 2; }
__device__ __forceinline__ uint32_t defl_lbase(uint32_t c)          // smallest length of code c
{
	if (c < 8u) return c + 3u;
	if (c == 28u) return 258u;
	const uint32_t e = (c - 4u) >> 2;
	return ((4u + (c & 3u)) << e) + 3u;
}
__device__ __forceinline__ uint32_t defl_dcode(uint32_t d)          // distance 1..32768 -> 0..29
{
	const uint32_t v = d - 1u;
	if (v < 4u) return v;
	const uint32_t e = 30u - __clz(v);                              // floor(log2 v) - 1
	return 2u * e + 2u + ((v >> e) & 1u);
}
__device__ __forceinline__ uint32_t defl_dextra(uint32_t c) { return c < 4u ? 0u : (c >> 1) - 1u; }
__device__ __forceinline__ uint32_t defl_dbase(uint32_t c)
{
	if (c < 4u) return c + 1u;
	const uint32_t e = (c >> 1) - 1u;
	return ((2u + (c & 1u)) << e) + 1u;
}
// the next piece of a match of L bytes (L >= 3): none longer than 258 or shorter than 3
__device__ __forceinline__ uint32_t match_piece(uint32_t L) { return L <= 258u ? L : L - 258u >= 3u ? 258u : L - 3u; }

// One LZ4 sequence of the block [b, b+clen) at *ip: literal count, match length (0 = the last sequence)
// and offset.  Every lane reads the same bytes.
__device__ __forceinline__ void lz4_seq(const uint8_t *b, uint32_t clen, uint32_t &ip, uint32_t &nl,
    uint32_t &ml, uint32_t &off)
{
	const uint32_t tok = b[ip++];
	nl = tok >> 4;
	if (nl == 15u) { uint32_t c; do { c = b[ip++]; nl += c; } while (c == 255u); }
	ip += nl;
	ml = 0; off = 0;
	if (ip >= clen) return;
	off = (uint32_t)b[ip] | ((uint32_t)b[ip + 1] << 8);
	ip += 2;
	ml = tok & 15u;
	if (ml == 15u) { uint32_t c; do { c = b[ip++]; ml += c; } while (c == 255u); }
	ml += 4u;
}

// Lengths of a length-limited huffman code of freq[0..n) into len[0..n) (tests/gzip_encode_ref.py
// huff_lengths): no used symbol -> all 0, one -> length 1; otherwise the used symbols sorted by
// (frequency, symbol), two-queue merge taking a leaf before an internal node of equal weight, length =
// depth; if the deepest leaf is deeper than `limit`, every used frequency f becomes (f + 1) / 2 and the
// code is built again.  Returns the number of used symbols.
__device__ uint32_t warp_huff_lengths(const uint32_t *freq, uint32_t n, uint32_t limit,
    uint8_t *len, DeflSmem &S, int lane)
{
	const uint32_t FULL = 0xffffffffu;
	uint32_t nu = 0;
	for (uint32_t b = 0; b < n; b += 32u) {
		const uint32_t s = b + (uint32_t)lane;
		const uint32_t f = s < n ? freq[s] : 0u;
		if (s < n) { S.w[s] = f; len[s] = 0; }
		nu += __popc(__ballot_sync(FULL, f != 0u));
	}
	__syncwarp();
	if (nu == 1u) {
		for (uint32_t s = (uint32_t)lane; s < n; s += 32u) if (S.w[s] != 0u) len[s] = 1;
		__syncwarp();
	}
	if (nu < 2u) return nu;
	for (;;) {
		// rank of each used symbol by (frequency, symbol)
		for (uint32_t s = (uint32_t)lane; s < n; s += 32u) {
			const uint32_t f = S.w[s];
			if (f == 0u) continue;
			uint32_t r = 0;
			for (uint32_t t = 0; t < n; t++) {
				const uint32_t g = S.w[t];
				r += g != 0u && (g < f || (g == f && t < s));
			}
			S.ord[r] = (uint16_t)s;
		}
		__syncwarp();
		if (lane == 0) {
			uint32_t i = 0, j = 0;
			for (uint32_t k = 0; k + 1u < nu; k++) {
				uint32_t w = 0;
#pragma unroll
				for (int q = 0; q < 2; q++) {
					const uint32_t lw = i < nu ? S.w[S.ord[i]] : 0u;
					if (i < nu && (j >= k || lw <= S.iw[j])) { S.lpar[i] = (uint16_t)k; w += lw; i++; }
					else { S.ipar[j] = (uint16_t)k; w += S.iw[j]; j++; }
				}
				S.iw[k] = w;
			}
			S.idep[nu - 2u] = 0;
			for (int k = (int)nu - 3; k >= 0; k--) S.idep[k] = (uint8_t)(S.idep[S.ipar[k]] + 1u);
		}
		__syncwarp();
		uint32_t mx = 0;
		for (uint32_t i = (uint32_t)lane; i < nu; i += 32u) mx = max(mx, (uint32_t)S.idep[S.lpar[i]] + 1u);
#pragma unroll
		for (int d = 16; d > 0; d >>= 1) mx = max(mx, __shfl_xor_sync(FULL, mx, d));
		if (mx <= limit) {
			for (uint32_t i = (uint32_t)lane; i < nu; i += 32u) len[S.ord[i]] = (uint8_t)(S.idep[S.lpar[i]] + 1u);
			__syncwarp();
			return nu;
		}
		for (uint32_t s = (uint32_t)lane; s < n; s += 32u) S.w[s] = (S.w[s] + 1u) >> 1;
		__syncwarp();
	}
}

// canonical codes of len[0..n) (RFC 1951 3.2.2), bit-reversed for LSB-first output: code | length << 16
__device__ __forceinline__ void warp_canon(const uint8_t *len, uint32_t n, uint32_t *code, DeflSmem &S, int lane)
{
	const uint32_t FULL = 0xffffffffu, lt = (1u << lane) - 1u;
	if (lane < 16) S.cnt[lane] = 0;
	__syncwarp();
	for (uint32_t b = 0; b < n; b += 32u) {
		const uint32_t s = b + (uint32_t)lane, L = s < n ? len[s] : 0u;
		const uint32_t m = __match_any_sync(FULL, L);
		if (L != 0u && (m & lt) == 0u) S.cnt[L] += (uint16_t)__popc(m);
		__syncwarp();
	}
	if (lane == 0) {
		uint32_t c = 0;
		for (uint32_t L = 1; L < 16u; L++) { c = (c + (L > 1u ? S.cnt[L - 1u] : 0u)) << 1; S.nxt[L] = c; }
	}
	__syncwarp();
	for (uint32_t b = 0; b < n; b += 32u) {
		const uint32_t s = b + (uint32_t)lane, L = s < n ? len[s] : 0u;
		const uint32_t m = __match_any_sync(FULL, L);
		const uint32_t c = L != 0u ? S.nxt[L] + (uint32_t)__popc(m & lt) : 0u;
		__syncwarp();
		if (L != 0u && (m & lt) == 0u) S.nxt[L] += (uint32_t)__popc(m);
		if (s < n) code[s] = L != 0u ? (rev16(c) >> (16u - L)) | (L << 16) : 0u;
		__syncwarp();
	}
}

// The bit writer: bits [0, bp) of S.buf are placed, S.buf[0] is output word `wo`.  One round places one
// item (v, n <= 32 bits, v < 2^n) per lane that has one, in lane order, and stores the completed words.
struct DeflOut {
	uint32_t *out;
	uint32_t wo, bp;
};
__device__ __forceinline__ void defl_put(DeflOut &o, DeflSmem &S, uint32_t v, uint32_t n, int lane)
{
	const uint32_t FULL = 0xffffffffu;
	uint32_t inc = n;
#pragma unroll
	for (int d = 1; d < 32; d <<= 1) {
		const uint32_t u = __shfl_up_sync(FULL, inc, d);
		if (lane >= d) inc += u;
	}
	const uint32_t tot = __shfl_sync(FULL, inc, 31);
	if (tot == 0u) return;
	const uint32_t p = o.bp + inc - n, sh = p & 31u;
	if (n != 0u) {
		atomicOr(&S.buf[p >> 5], v << sh);
		if (sh + n > 32u) atomicOr(&S.buf[(p >> 5) + 1u], v >> (32u - sh));
	}
	__syncwarp();
	o.bp += tot;
	const uint32_t full = o.bp >> 5;
	if (full != 0u) {
		for (uint32_t i = (uint32_t)lane; i < full; i += 32u) o.out[o.wo + i] = S.buf[i];
		const uint32_t carry = S.buf[full];
		__syncwarp();
		for (uint32_t i = (uint32_t)lane; i < DEFL_BUFW; i += 32u) S.buf[i] = i == 0u ? carry : 0u;
		__syncwarp();
		o.wo += full; o.bp &= 31u;
	}
}

// Gathers the items of walk 2 into rounds of 32: lane k holds the round's k-th item.
struct DeflRound {
	uint32_t v, n, fill;
};
__device__ __forceinline__ void round_flush(DeflRound &r, DeflOut &o, DeflSmem &S, int lane)
{
	defl_put(o, S, r.v, r.n, lane);
	r.v = 0; r.n = 0; r.fill = 0;
}
// the literal symbols of src[0, k)
__device__ __forceinline__ void round_lits(DeflRound &r, DeflOut &o, DeflSmem &S, const uint8_t *src, uint32_t k, int lane)
{
	while (k != 0u) {
		const uint32_t t = min(k, 32u - r.fill);
		const uint32_t i = (uint32_t)lane - r.fill;
		if ((uint32_t)lane >= r.fill && i < t) {
			const uint32_t c = S.lf[src[i]];
			r.v = c & 0xffffu; r.n = c >> 16;
		}
		r.fill += t; src += t; k -= t;
		if (r.fill == 32u) round_flush(r, o, S, lane);
	}
}
// one match piece of length L at distance d: two items
__device__ __forceinline__ void round_match(DeflRound &r, DeflOut &o, DeflSmem &S, uint32_t L, uint32_t d, int lane)
{
	if (r.fill > 30u) round_flush(r, o, S, lane);
	const uint32_t lc = defl_lcode(L), dc = defl_dcode(d);
	if ((uint32_t)lane == r.fill) {
		const uint32_t c = S.lf[257u + lc];
		r.v = (c & 0xffffu) | ((L - defl_lbase(lc)) << (c >> 16)); r.n = (c >> 16) + defl_lextra(lc);
	} else if ((uint32_t)lane == r.fill + 1u) {
		const uint32_t c = S.df[dc];
		r.v = (c & 0xffffu) | ((d - defl_dbase(dc)) << (c >> 16)); r.n = (c >> 16) + defl_dextra(dc);
	}
	r.fill += 2u;
	if (r.fill == 32u) round_flush(r, o, S, lane);
}

// The zlib frame of one record.  `src` logical bytes (lsize), `lz` K3's frame (BE32 clen + block).
// Returns the padded frame size when it is smaller than `limit` and then writes it at `out` (4-byte
// aligned); otherwise writes nothing and returns lsize.
__device__ __forceinline__ uint32_t warp_deflate_from_lz4(const uint8_t *__restrict__ src, uint32_t lsize,
    const uint8_t *lz, uint32_t limit, uint32_t *out, DeflSmem &S, int lane)
{
	const uint32_t FULL = 0xffffffffu;
	const uint32_t clen = ((uint32_t)lz[0] << 24) | ((uint32_t)lz[1] << 16) | ((uint32_t)lz[2] << 8) | lz[3];
	const uint8_t *blk = lz + 4;
	// ---- walk 1: histograms
	for (uint32_t i = (uint32_t)lane; i < 288u; i += 32u) S.lf[i] = 0;
	if (lane < 32) S.df[lane] = 0;
	if (lane < 20) S.cf[lane] = 0;
	__syncwarp();
	uint32_t nmatch = 0;
	{
		uint32_t ip = 0, pos = 0;
		while (ip < clen) {
			uint32_t nl, ml, off;
			lz4_seq(blk, clen, ip, nl, ml, off);
			for (uint32_t i = (uint32_t)lane; i < nl; i += 32u) atomicAdd(&S.lf[src[pos + i]], 1u);
			pos += nl;
			if (ml == 0u) break;
			if (off > DEFL_MAXDIST) {
				for (uint32_t i = (uint32_t)lane; i < ml; i += 32u) atomicAdd(&S.lf[src[pos + i]], 1u);
			} else {
				const uint32_t dc = defl_dcode(off);
				for (uint32_t L = ml; L != 0u; ) {
					const uint32_t p = match_piece(L);
					if (lane == 0) { S.lf[257u + defl_lcode(p)]++; S.df[dc]++; }
					nmatch++; L -= p;
				}
			}
			pos += ml;
		}
	}
	if (lane == 0) S.lf[256] = 1;
	__syncwarp();
	// ---- the codes
	warp_huff_lengths(S.lf, 286u, 15u, S.len, S, lane);
	if (nmatch == 0u) {
		if (lane < 30) S.len[288 + lane] = lane == 0 ? 1u : 0u;
		__syncwarp();
	} else {
		warp_huff_lengths(S.df, 30u, 15u, S.len + 288, S, lane);
	}
	uint32_t hlit = 257u, hdist = 1u;
	for (uint32_t s = (uint32_t)lane; s < 286u; s += 32u) if (S.len[s]) hlit = max(hlit, s + 1u);
	if (lane < 30 && S.len[288 + lane]) hdist = max(hdist, (uint32_t)lane + 1u);
#pragma unroll
	for (int d = 16; d > 0; d >>= 1) {
		hlit = max(hlit, __shfl_xor_sync(FULL, hlit, d));
		hdist = max(hdist, __shfl_xor_sync(FULL, hdist, d));
	}
	// the code-length symbols (serial, at most hlit + hdist of them)
	uint32_t ncls = 0;
	if (lane == 0) {
		const uint32_t n = hlit + hdist;
		auto at = [&](uint32_t i) -> uint32_t { return i < hlit ? S.len[i] : S.len[288u + i - hlit]; };
		uint32_t i = 0;
		while (i < n) {
			const uint32_t v = at(i);
			uint32_t r = 1;
			while (i + r < n && at(i + r) == v) r++;
			if (v == 0u && r >= 3u) {
				const uint32_t k = min(r, 138u);
				const uint32_t s = k >= 11u ? 18u : 17u, x = k >= 11u ? k - 11u : k - 3u;
				S.cls[ncls++] = (uint16_t)(s | (x << 5)); S.cf[s]++;
				i += k;
				continue;
			}
			S.cls[ncls++] = (uint16_t)v; S.cf[v]++;
			i++; r--;
			while (v != 0u && r >= 3u) {
				const uint32_t k = min(r, 6u);
				S.cls[ncls++] = (uint16_t)(16u | ((k - 3u) << 5)); S.cf[16]++;
				i += k; r -= k;
			}
		}
	}
	ncls = __shfl_sync(FULL, ncls, 0);
	__syncwarp();
	warp_huff_lengths(S.cf, 19u, 7u, S.clen, S, lane);
	// RFC 1951 3.2.7: the order of the code-length code's lengths
	const uint32_t my_cl = lane < 19 ? (lane == 0 ? 16u : lane == 1 ? 17u : lane == 2 ? 18u : lane == 3 ? 0u :
	    ((lane - 4) & 1) ? 7u - (uint32_t)(lane - 4) / 2u : 8u + (uint32_t)(lane - 4) / 2u) : 0u;
	const uint32_t my_cll = lane < 19 ? S.clen[my_cl] : 0u;
	const uint32_t hclen = max(4u, 32u - __clz(__ballot_sync(FULL, my_cll != 0u)));
	// code sizes, before the frequency arrays become code tables
	uint64_t bits = 0;
	for (uint32_t s = (uint32_t)lane; s < 286u; s += 32u)
		bits += (uint64_t)S.lf[s] * (S.len[s] + (s >= 257u ? defl_lextra(s - 257u) : 0u));
	if (lane < 30) bits += (uint64_t)S.df[lane] * (S.len[288 + lane] + defl_dextra((uint32_t)lane));
	if (lane < 19) bits += (uint64_t)S.cf[lane] * (S.clen[lane] + (lane == 16 ? 2u : lane == 17 ? 3u : lane == 18 ? 7u : 0u));
#pragma unroll
	for (int d = 16; d > 0; d >>= 1) bits += __shfl_xor_sync(FULL, bits, d);
	bits += 17u + 3u * hclen;                                       // block header
	const uint64_t bytes = 2ull + (bits + 7u) / 8u + 4ull;
	const uint64_t padded = (bytes + 511u) & ~511ull;
	if (padded >= limit) return lsize;
	__syncwarp();
	warp_canon(S.len, 286u, S.lf, S, lane);
	warp_canon(S.len + 288, 30u, S.df, S, lane);
	warp_canon(S.clen, 19u, S.cf, S, lane);
	// ---- walk 2: the bits
	for (uint32_t i = (uint32_t)lane; i < DEFL_BUFW; i += 32u) S.buf[i] = 0;
	__syncwarp();
	DeflOut o; o.out = out; o.wo = 0; o.bp = 0;
	defl_put(o, S, lane == 0 ? 0x0178u : 5u | ((hlit - 257u) << 3) | ((hdist - 1u) << 8) | ((hclen - 4u) << 13),
	    lane == 0 ? 16u : lane == 1 ? 17u : 0u, lane);
	defl_put(o, S, my_cll, (uint32_t)lane < hclen ? 3u : 0u, lane);
	for (uint32_t b = 0; b < ncls; b += 32u) {
		const uint32_t i = b + (uint32_t)lane;
		uint32_t v = 0, n = 0;
		if (i < ncls) {
			const uint32_t e = S.cls[i], s = e & 31u, c = S.cf[s];
			v = (c & 0xffffu) | ((e >> 5) << (c >> 16));
			n = (c >> 16) + (s == 16u ? 2u : s == 17u ? 3u : s == 18u ? 7u : 0u);
		}
		defl_put(o, S, v, n, lane);
	}
	{
		DeflRound r; r.v = 0; r.n = 0; r.fill = 0;
		uint32_t ip = 0, pos = 0;
		while (ip < clen) {
			uint32_t nl, ml, off;
			lz4_seq(blk, clen, ip, nl, ml, off);
			round_lits(r, o, S, src + pos, nl, lane);
			pos += nl;
			if (ml == 0u) break;
			if (off > DEFL_MAXDIST) {
				round_lits(r, o, S, src + pos, ml, lane);
			} else {
				for (uint32_t L = ml; L != 0u; ) {
					const uint32_t p = match_piece(L);
					round_match(r, o, S, p, off, lane);
					L -= p;
				}
			}
			pos += ml;
		}
		if (r.fill == 32u) round_flush(r, o, S, lane);
		if ((uint32_t)lane == r.fill) { r.v = S.lf[256] & 0xffffu; r.n = S.lf[256] >> 16; }
		round_flush(r, o, S, lane);
	}
	const uint32_t pad = (8u - (o.bp & 7u)) & 7u;
	const uint32_t ad = warp_adler32(src, lsize, lane);
	const uint32_t be = (ad >> 24) | ((ad >> 8) & 0xff00u) | ((ad << 8) & 0xff0000u) | (ad << 24);
	defl_put(o, S, lane == 0 ? 0u : be, lane == 0 ? pad : lane == 1 ? 32u : 0u, lane);
	// the last partial word and the zero padding
	const uint32_t nw = (uint32_t)(padded / 4u);
	for (uint32_t i = o.wo + (uint32_t)lane; i < nw; i += 32u) out[i] = i == o.wo ? S.buf[0] : 0u;
	__syncwarp();
	return (uint32_t)padded;
}

// One warp per job (grid-stride) of `enc`, K3's jobs after K3: a record K3 stored as an LZ4 frame (out_len <
// lsize) is re-coded from that frame.  Logical bytes at src_base + src_off, the LZ4 frame at lz_base +
// dst_off, the zlib frame written at gz_base + dst_off.  `vs_enc`: the frame is written only when its
// padded size is smaller than K3's (COMPRESS), otherwise when it is smaller than lsize
// (mtz_k_gzip_encode).  gz[j].out_len = the padded size, or lsize when no frame was written; when gz
// is not enc, gz[j] is enc[j] with dst_off = the frame's address (k_layout / k_assemble read it).
__global__ void __launch_bounds__(DEFL_THREADS)
k_deflate_from_lz4(const mtz_job *enc, mtz_job *gz, uint32_t njobs, uint64_t src_base, uint64_t lz_base,
    uint64_t gz_base, bool vs_enc)
{
	__shared__ DeflSmem s_w[DEFL_WARPS];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t gw = blockIdx.x * DEFL_WARPS + (uint32_t)warp;
	const uint32_t nw = gridDim.x * DEFL_WARPS;
	for (uint32_t j = gw; j < njobs; j += nw) {
		const mtz_job e = enc[j];
		uint32_t ol = e.lsize;
		if (e.lsize != 0u && e.out_len < e.lsize)
			ol = warp_deflate_from_lz4(reinterpret_cast<const uint8_t *>((uintptr_t)(src_base + e.src_off)), e.lsize,
			    reinterpret_cast<const uint8_t *>((uintptr_t)(lz_base + e.dst_off)), vs_enc ? e.out_len : e.lsize,
			    reinterpret_cast<uint32_t *>((uintptr_t)(gz_base + e.dst_off)), s_w[warp], lane);
		__syncwarp();
		if (lane == 0) {
			if (gz != enc) {
				mtz_job g = e;
				g.dst_off = gz_base + e.dst_off; g.out_len = ol; g.status = MTZ_OK;
				gz[j] = g;
			} else {
				gz[j].out_len = ol; gz[j].status = MTZ_OK;
			}
		}
	}
}

} // namespace mtz
