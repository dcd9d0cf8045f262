// fletcher.cuh -- K1: Fletcher-4 partial sums on sm_90a (integer, HBM-bound).
//
// The arithmetic replaced here runs today inside the `zfs send` / `zfs recv`
// children that the reference spawns (lib/backupSender.js:177,
// lib/zfsClient.js:793): fletcher_4 over every stream byte.  SURVEY.md App. A.2.
//
// fletcher_4 is a serial recurrence (a+=w; b+=a; c+=b; d+=c).  Its closed form
// over a segment of n words, with k = 1-based distance of a word from the END:
//     A = sum w   B = sum k w   C = sum T2(k) w   D = sum T3(k) w   (mod 2^64)
// T2(k)=k(k+1)/2, T3(k)=k(k+1)(k+2)/6.  A warp walks the segment in 512-byte
// rows (32 lanes x 16 B, fully coalesced LDG.128).  With m = row index counted
// from the end, lane t element e holds word k = 128 m + delta,
// delta = q - (4t+e).  Each lane keeps, per element, the four sums over rows
//     sa = sum w, sb = sum m w, sc = sum T2(m) w, sd = sum T3(m) w
// (one 32x32+64 IMAD.WIDE each: the row weights are warp-uniform 32-bit
// values), and converts them to the k-basis once per chunk with the Newton
// forward-difference identity for the integer-valued polynomials
// T2(128m+delta), T3(128m+delta) in the basis {1, m, T2(m), T3(m)} -- integer
// coefficients, hence exact mod 2^64 with no division.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

namespace mtz {

struct Ck4 { uint64_t a, b, c, d; };
// n = word count; bit 63 of n (PART_RESET) marks a segment that begins with a
// DRR_BEGIN record: the stream checksum restarts there, so whatever precedes
// the segment is ignored (segmented scan).
struct Part { uint64_t n, a, b, c, d; };
#define PART_RESET (1ull << 63)
#define PART_NMASK (~PART_RESET)

__host__ __device__ __forceinline__ uint64_t tri2(uint64_t n)
{
	uint64_t x = n, y = n + 1;
	if (x & 1) y >>= 1; else x >>= 1;
	return x * y;
}

// n < 2^32 fast paths: 32-bit remainder instead of a 64-bit division
__host__ __device__ __forceinline__ uint64_t tri3_u32(uint32_t n)
{
	uint64_t f0 = n, f1 = (uint64_t)n + 1, f2 = (uint64_t)n + 2;
	if (!(n & 1u)) f0 >>= 1; else f1 >>= 1;
	const uint32_t r = n % 3u;                     // n%3==0 -> f0, 2 -> f1, 1 -> f2
	if (r == 0u) f0 /= 3u; else if (r == 2u) f1 /= 3u; else f2 /= 3u;
	return f0 * f1 * f2;
}

__host__ __device__ __forceinline__ uint64_t tri3(uint64_t n)
{
	if (n < 0xfffffff0ull) return tri3_u32((uint32_t)n);
	uint64_t f0 = n, f1 = n + 1, f2 = n + 2;
	if (!(f0 & 1)) f0 >>= 1; else f1 >>= 1;          // one of n, n+1 is even
	if (f0 % 3 == 0) f0 /= 3; else if (f1 % 3 == 0) f1 /= 3; else f2 /= 3;
	return f0 * f1 * f2;
}

// running state (a,b,c,d) followed by a segment whose zero-state sums are p
__host__ __device__ __forceinline__ Ck4 apply(const Ck4 &s0, const Part &p)
{
	const uint64_t n = p.n & PART_NMASK, t2 = tri2(n), t3 = tri3(n);
	Ck4 s = s0;
	if (p.n & PART_RESET) s.a = s.b = s.c = s.d = 0;
	Ck4 r;
	r.a = s.a + p.a;
	r.b = s.b + n * s.a + p.b;
	r.c = s.c + n * s.b + t2 * s.a + p.c;
	r.d = s.d + n * s.c + t2 * s.b + t3 * s.a + p.d;
	return r;
}

__host__ __device__ __forceinline__ Part concat(const Part &x, const Part &y)
{
	if (y.n & PART_RESET) return y;
	Ck4 s = { x.a, x.b, x.c, x.d };
	s = apply(s, y);
	Part r = { x.n + y.n, s.a, s.b, s.c, s.d };    // x's reset bit carries over
	return r;
}

// fold the 8 little-endian u32 words of a zio_cksum_t value into the state
__host__ __device__ __forceinline__ Ck4 fold_cksum_words(Ck4 s, const Ck4 &v)
{
	const uint64_t q[4] = { v.a, v.b, v.c, v.d };
#pragma unroll
	for (int i = 0; i < 4; i++) {
		s.a += (uint32_t)q[i];         s.b += s.a; s.c += s.b; s.d += s.c;
		s.a += (uint32_t)(q[i] >> 32); s.b += s.a; s.c += s.b; s.d += s.c;
	}
	return s;
}

#ifdef __CUDACC__

#ifndef K1_UNROLL
#define K1_UNROLL 12          // LDG.128 in flight per lane
#endif

__device__ __forceinline__ uint4 ldg_stream(const uint4 *p)
{
#ifdef MTZ_HOST_EMUL      // tests/emul compiles this header for the CPU warp emulator
	return *p;
#else
	uint4 r;
	asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
	    : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
	return r;
#endif
}

__device__ __forceinline__ uint64_t shfl_xor64(uint64_t v, int m)
{
	uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
	lo = __shfl_xor_sync(0xffffffffu, lo, m);
	hi = __shfl_xor_sync(0xffffffffu, hi, m);
	return ((uint64_t)hi << 32) | lo;
}

__device__ __forceinline__ uint64_t warp_sum64(uint64_t v)
{
#pragma unroll
	for (int m = 16; m > 0; m >>= 1) v += shfl_xor64(v, m);
	return v;
}

struct RowAcc {
	uint64_t sa[4], sb[4], sc[4], sd[4];
	__device__ __forceinline__ void zero()
	{
#pragma unroll
		for (int e = 0; e < 4; e++) sa[e] = sb[e] = sc[e] = sd[e] = 0;
	}
	__device__ __forceinline__ void add(const uint4 &v, uint32_t m, uint32_t t2,
	    uint32_t t3)
	{
		const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
		for (int e = 0; e < 4; e++) {
			sa[e] += w[e];
			sb[e] += (uint64_t)w[e] * m;
			sc[e] += (uint64_t)w[e] * t2;
			sd[e] += (uint64_t)w[e] * t3;
		}
	}
};

// Maximum rows one call may cover: T3(m) must fit 32 bits (m <= 2952).
#define MTZ_K1_MAX_ROWS 2048u

// Warp-cooperative zero-state sums of the words in [p0, p0 + 4*nwords).
// p0 is 4-byte aligned; every 16-byte vector that intersects the segment must
// be readable (buffers are 16-byte aligned and padded).  All lanes return the
// same (A,B,C,D).  Requires rows <= MTZ_K1_MAX_ROWS.
__device__ __forceinline__ Ck4 warp_fletcher(const uint8_t *p0, uint32_t nwords,
    int lane)
{
	Ck4 out = { 0, 0, 0, 0 };
	if (nwords == 0) return out;
	const uintptr_t a0 = (uintptr_t)p0;
	const uintptr_t abase = a0 & ~(uintptr_t)511;
	const uint32_t head = (uint32_t)((a0 - abase) >> 2);   // words skipped in row 0
	const uint32_t E = head + nwords;                       // words abase..end
	const uint32_t NR = (E + 127u) >> 7;
	const uint32_t q = E - 128u * (NR - 1u);               // 1..128 words in last row
	const uint4 *rowp = reinterpret_cast<const uint4 *>(abase) + lane;
	const uint32_t r0 = 4u * (uint32_t)lane;

	RowAcc acc; acc.zero();
	uint32_t m = NR - 1u;
	uint32_t t2 = (m * (m + 1u)) >> 1;
	uint32_t t3 = (uint32_t)(((uint64_t)m * (m + 1u) * (m + 2u)) / 6u);

	// ---- first row (head mask; also tail mask when it is the only row) ----
	{
		uint4 v = make_uint4(0, 0, 0, 0);
		const uint32_t lim = (NR == 1u) ? q : 128u;
		if (r0 + 4u > head && r0 < lim) {
			v = ldg_stream(rowp);
			if (r0 + 0u < head || r0 + 0u >= lim) v.x = 0;
			if (r0 + 1u < head || r0 + 1u >= lim) v.y = 0;
			if (r0 + 2u < head || r0 + 2u >= lim) v.z = 0;
			if (r0 + 3u < head || r0 + 3u >= lim) v.w = 0;
		}
		acc.add(v, m, t2, t3);
	}
	if (NR > 1u) {
		// ---- full middle rows j = 1 .. NR-2, four loads in flight ----
		uint32_t j = 1u;
		const uint32_t jend = NR - 1u;
		for (; j + K1_UNROLL <= jend; j += K1_UNROLL) {
			uint4 v[K1_UNROLL];
#pragma unroll
			for (int u = 0; u < K1_UNROLL; u++) v[u] = ldg_stream(rowp + 32u * (j + (uint32_t)u));
#pragma unroll
			for (int u = 0; u < K1_UNROLL; u++) {
				t3 -= t2; t2 -= m; m -= 1u; acc.add(v[u], m, t2, t3);
			}
		}
		for (; j + 4u <= jend; j += 4u) {
			uint4 v0 = ldg_stream(rowp + 32u * (j + 0u));
			uint4 v1 = ldg_stream(rowp + 32u * (j + 1u));
			uint4 v2 = ldg_stream(rowp + 32u * (j + 2u));
			uint4 v3 = ldg_stream(rowp + 32u * (j + 3u));
			t3 -= t2; t2 -= m; m -= 1u; acc.add(v0, m, t2, t3);
			t3 -= t2; t2 -= m; m -= 1u; acc.add(v1, m, t2, t3);
			t3 -= t2; t2 -= m; m -= 1u; acc.add(v2, m, t2, t3);
			t3 -= t2; t2 -= m; m -= 1u; acc.add(v3, m, t2, t3);
		}
		for (; j < jend; j++) {
			uint4 v = ldg_stream(rowp + 32u * j);
			t3 -= t2; t2 -= m; m -= 1u; acc.add(v, m, t2, t3);
		}
		// ---- last row (m == 0): only sa matters, tail mask ----
		{
			uint4 v = make_uint4(0, 0, 0, 0);
			if (r0 < q) {
				v = ldg_stream(rowp + 32u * jend);
				if (r0 + 1u >= q) v.y = 0;
				if (r0 + 2u >= q) v.z = 0;
				if (r0 + 3u >= q) v.w = 0;
			}
			acc.add(v, 0u, 0u, 0u);
		}
	}

	// ---- row basis -> word-distance basis, per element ----
	// Q(i) = T2(128 i + d), P(i) = T3(128 i + d); |128 i + d| < 600 so every
	// product fits int32 and the divisions are by constants.
#pragma unroll
	for (int e = 0; e < 4; e++) {
		const int d = (int)q - (int)(r0 + (uint32_t)e);
		const int Q0 = d * (d + 1) / 2;
		const int Q1 = (d + 128) * (d + 129) / 2;
		int P[4];
#pragma unroll
		for (int i = 0; i < 4; i++) {
			const int x = d + 128 * i;
			P[i] = x * (x + 1) * (x + 2) / 6;
		}
		const int q2 = 16384;
		const int q1 = Q1 - Q0;
		const int d1 = P[1] - P[0];
		const int d2 = P[2] - 2 * P[1] + P[0];
		const int d3 = 2097152;                       // 128^3
		const uint64_t sa = acc.sa[e], sb = acc.sb[e], sc = acc.sc[e], sd = acc.sd[e];
		out.a += sa;
		out.b += 128ull * sb + (uint64_t)(int64_t)d * sa;
		out.c += (uint64_t)q2 * sc + (uint64_t)(int64_t)(q1 - q2) * sb + (uint64_t)(int64_t)Q0 * sa;
		out.d += (uint64_t)d3 * sd + (uint64_t)(int64_t)(d2 - 2 * d3) * sc +
		    (uint64_t)(int64_t)(d1 - d2 + d3) * sb + (uint64_t)(int64_t)P[0] * sa;
	}
	out.a = warp_sum64(out.a);
	out.b = warp_sum64(out.b);
	out.c = warp_sum64(out.c);
	out.d = warp_sum64(out.d);
	return out;
}

// ---------------------------------------------------------------------------
// Group form of the same computation: G = 8, 16 or 32 lanes own one segment
// (rows of 16*G bytes), so a warp works on 32/G small records at once and the
// fixed cost per record (basis conversion, reduction) is shared.  Everything is
// identical to warp_fletcher with 128 replaced by RW = 4*G words per row; the
// shuffles of the final reduction stay inside the group (xor masks < G).
template <int G>
__device__ __forceinline__ Ck4 group_fletcher(const uint8_t *p0, uint32_t nwords, int gl)
{
	constexpr uint32_t RW = 4u * G;                 // words per row
	constexpr uint32_t RB = 16u * G;                // bytes per row
	Ck4 out = { 0, 0, 0, 0 };
	RowAcc acc; acc.zero();
	uint32_t q = 1;
	if (nwords != 0u) {
		const uintptr_t a0 = (uintptr_t)p0;
		const uintptr_t abase = a0 & ~(uintptr_t)(RB - 1u);
		const uint32_t head = (uint32_t)((a0 - abase) >> 2);
		const uint32_t E = head + nwords;
		const uint32_t NR = (E + RW - 1u) / RW;
		q = E - RW * (NR - 1u);                      // 1..RW words in the last row
		const uint4 *rowp = reinterpret_cast<const uint4 *>(abase) + gl;
		const uint32_t r0 = 4u * (uint32_t)gl;
		uint32_t m = NR - 1u;
		uint32_t t2 = (m * (m + 1u)) >> 1;
		uint32_t t3 = (uint32_t)(((uint64_t)m * (m + 1u) * (m + 2u)) / 6u);
		{
			uint4 v = make_uint4(0, 0, 0, 0);
			const uint32_t lim = (NR == 1u) ? q : RW;
			if (r0 + 4u > head && r0 < lim) {
				v = ldg_stream(rowp);
				if (r0 + 0u < head || r0 + 0u >= lim) v.x = 0;
				if (r0 + 1u < head || r0 + 1u >= lim) v.y = 0;
				if (r0 + 2u < head || r0 + 2u >= lim) v.z = 0;
				if (r0 + 3u < head || r0 + 3u >= lim) v.w = 0;
			}
			acc.add(v, m, t2, t3);
		}
		if (NR > 1u) {
			uint32_t j = 1u;
			const uint32_t jend = NR - 1u;
			for (; j + K1_UNROLL <= jend; j += K1_UNROLL) {
				uint4 v[K1_UNROLL];
#pragma unroll
				for (int u = 0; u < K1_UNROLL; u++) v[u] = ldg_stream(rowp + (uint32_t)G * (j + (uint32_t)u));
#pragma unroll
				for (int u = 0; u < K1_UNROLL; u++) {
					t3 -= t2; t2 -= m; m -= 1u; acc.add(v[u], m, t2, t3);
				}
			}
			for (; j + 4u <= jend; j += 4u) {
				uint4 v0 = ldg_stream(rowp + (uint32_t)G * (j + 0u));
				uint4 v1 = ldg_stream(rowp + (uint32_t)G * (j + 1u));
				uint4 v2 = ldg_stream(rowp + (uint32_t)G * (j + 2u));
				uint4 v3 = ldg_stream(rowp + (uint32_t)G * (j + 3u));
				t3 -= t2; t2 -= m; m -= 1u; acc.add(v0, m, t2, t3);
				t3 -= t2; t2 -= m; m -= 1u; acc.add(v1, m, t2, t3);
				t3 -= t2; t2 -= m; m -= 1u; acc.add(v2, m, t2, t3);
				t3 -= t2; t2 -= m; m -= 1u; acc.add(v3, m, t2, t3);
			}
			for (; j < jend; j++) {
				uint4 v = ldg_stream(rowp + (uint32_t)G * j);
				t3 -= t2; t2 -= m; m -= 1u; acc.add(v, m, t2, t3);
			}
			{
				uint4 v = make_uint4(0, 0, 0, 0);
				if (r0 < q) {
					v = ldg_stream(rowp + (uint32_t)G * jend);
					if (r0 + 1u >= q) v.y = 0;
					if (r0 + 2u >= q) v.z = 0;
					if (r0 + 3u >= q) v.w = 0;
				}
				acc.add(v, 0u, 0u, 0u);
			}
		}
	}
	// row basis -> word-distance basis: k = RW * m + d
#pragma unroll
	for (int e = 0; e < 4; e++) {
		const int d = (int)q - (int)(4u * (uint32_t)gl + (uint32_t)e);
		const int Q0 = d * (d + 1) / 2;
		const int Q1 = (d + (int)RW) * (d + (int)RW + 1) / 2;
		int P[4];
#pragma unroll
		for (int i = 0; i < 4; i++) {
			const int x = d + (int)RW * i;
			P[i] = x * (x + 1) * (x + 2) / 6;
		}
		const int q2 = (int)(RW * RW);
		const int q1 = Q1 - Q0;
		const int d1 = P[1] - P[0];
		const int d2 = P[2] - 2 * P[1] + P[0];
		const int d3 = (int)(RW * RW * RW);
		const uint64_t sa = acc.sa[e], sb = acc.sb[e], sc = acc.sc[e], sd = acc.sd[e];
		out.a += sa;
		out.b += (uint64_t)RW * sb + (uint64_t)(int64_t)d * sa;
		out.c += (uint64_t)q2 * sc + (uint64_t)(int64_t)(q1 - q2) * sb + (uint64_t)(int64_t)Q0 * sa;
		out.d += (uint64_t)d3 * sd + (uint64_t)(int64_t)(d2 - 2 * d3) * sc +
		    (uint64_t)(int64_t)(d1 - d2 + d3) * sb + (uint64_t)(int64_t)P[0] * sa;
	}
#pragma unroll
	for (int mk = G / 2; mk > 0; mk >>= 1) {
		out.a += shfl_xor64(out.a, mk); out.b += shfl_xor64(out.b, mk);
		out.c += shfl_xor64(out.c, mk); out.d += shfl_xor64(out.d, mk);
	}
	return out;
}

// sums of the 70 header words [0,280) computed directly (k = 70 - index is tiny, so
// the products are plain 64-bit): the group's lanes take words gl, gl+G, ...
template <int G>
__device__ __forceinline__ Ck4 group_head70(const uint8_t *hdr, int gl)
{
	Ck4 o = { 0, 0, 0, 0 };
	const uint32_t *w = reinterpret_cast<const uint32_t *>(hdr);
	for (uint32_t i = (uint32_t)gl; i < 70u; i += (uint32_t)G) {
		const uint64_t v = w[i];
		const uint64_t k = 70u - i;
		o.a += v;
		o.b += k * v;
		o.c += (k * (k + 1u) / 2u) * v;
		o.d += (k * (k + 1u) * (k + 2u) / 6u) * v;
	}
#pragma unroll
	for (int mk = G / 2; mk > 0; mk >>= 1) {
		o.a += shfl_xor64(o.a, mk); o.b += shfl_xor64(o.b, mk);
		o.c += shfl_xor64(o.c, mk); o.d += shfl_xor64(o.d, mk);
	}
	return o;
}

// sums of a chunk followed by z zero words (moves the chunk's reference point)
__device__ __forceinline__ Ck4 shift_zeros(const Ck4 &p, uint64_t z)
{
	const uint64_t t2 = tri2(z), t3 = tri3(z);
	Ck4 r;
	r.a = p.a;
	r.b = p.b + z * p.a;
	r.c = p.c + z * p.b + t2 * p.a;
	r.d = p.d + z * p.c + t2 * p.b + t3 * p.a;
	return r;
}

#endif // __CUDACC__
} // namespace mtz
