// kernels_sha256.cuh -- block checksums with SHA-256 keys (MTZ_FLAG_BLOCK_SHA256): the records
// k_block_check leaves alone because their drr_checksumtype is 8 ([EXTERNAL] ZIO_CHECKSUM_SHA256,
// the setting dedup and nopwrite require).  Same table (block_classify), same bytes, same zero
// extension to the covered size, same verdicts; only the hash differs.
//
// Key format ([EXTERNAL] OpenZFS zio_checksum_SHA256 / abd_checksum_sha256): the 32-byte FIPS 180-4
// digest d of the PSIZE (or LSIZE) bytes the key covers is stored as
//   ddk_cksum.zc_word[i] = BE_64(d[8i .. 8i+8))
// and the words travel in the stream as native little-endian u64, so word i = (H[2i] << 32) | H[2i+1]
// with H the eight state words of the final hash.  The message is a multiple of 512 bytes: its
// padding is always one extra 64-byte block.
//
// SHA-256 is serial within a message, so the parallelism is across records: one thread per record,
// a warp hashes 32 records in lockstep.  The message schedule is a rolling 16-word window in
// registers, the round loop is unrolled (the constants fold into immediates), rotations are
// funnel shifts, Ch / Maj / three-way xors are left to LOP3.  The next 64-byte block is loaded while
// the current one compresses.
#pragma once
#include "kernels_block.cuh"

namespace mtz {

// round constant t; called with a constant t in the unrolled round loop, so it folds to an immediate
__device__ __forceinline__ uint32_t sha256_k(int t)
{
	const uint32_t k[64] = {
		0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
		0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
		0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
		0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
		0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
		0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
		0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
		0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u,
	};
	return k[t];
}

__device__ __forceinline__ uint32_t sha_rotr(uint32_t x, uint32_t n) { return __funnelshift_r(x, x, n); }
// byte swap (one PRMT)
__device__ __forceinline__ uint32_t sha_be32(uint32_t x)
{
	return (x >> 24) | ((x >> 8) & 0xff00u) | ((x << 8) & 0xff0000u) | (x << 24);
}

// FIPS 180-4 SHA-256 compression of one 64-byte block (`w` = its 16 big-endian words, consumed)
__device__ __forceinline__ void sha256_compress(uint32_t st[8], uint32_t w[16])
{
	uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
	for (int t = 0; t < 64; t++) {
		if (t >= 16) {
			const uint32_t x = w[(t - 15) & 15], y = w[(t - 2) & 15];
			const uint32_t s0 = sha_rotr(x, 7) ^ sha_rotr(x, 18) ^ (x >> 3);
			const uint32_t s1 = sha_rotr(y, 17) ^ sha_rotr(y, 19) ^ (y >> 10);
			w[t & 15] += s0 + w[(t - 7) & 15] + s1;
		}
		const uint32_t t1 = h + (sha_rotr(e, 6) ^ sha_rotr(e, 11) ^ sha_rotr(e, 25)) + ((e & f) ^ (~e & g)) +
		    sha256_k(t) + w[t & 15];
		const uint32_t t2 = (sha_rotr(a, 2) ^ sha_rotr(a, 13) ^ sha_rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
		h = g; g = f; f = e; e = d + t1;
		d = c; c = b; b = a; a = t1 + t2;
	}
	st[0] += a; st[1] += b; st[2] += c; st[3] += d;
	st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

__device__ __forceinline__ uint64_t sha_join(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }
// the big-endian u64 of 8 bytes loaded as a little-endian uint2 (also: bswap64 of sha_join(x, y))
__device__ __forceinline__ uint64_t sha_be64(uint2 v) { return sha_join(sha_be32(v.y), sha_be32(v.x)); }

// Block k of the message "nbytes of `p`, zeros up to `cover`, FIPS 180-4 padding" as 16 big-endian
// words W: SHA-256's 64-byte blocks of 32-bit words, SHA-512's 128-byte blocks of 64-bit words.
// `p` is 8-byte aligned, `nbytes` a multiple of 8, `cover` a multiple of the block; no byte at or
// past p[nbytes] is read (the zeros are arithmetic).
template <class W>
__device__ __forceinline__ void sha_message_block(const uint8_t *__restrict__ p, uint64_t nbytes,
    uint64_t cover, uint64_t k, W w[16])
{
	constexpr uint64_t block = 16 * sizeof(W);
	const uint64_t o = k * block;
	auto put = [&](int i, uint2 v) {      // chunk i: 8 bytes
		if constexpr (sizeof(W) == 4) {
			w[2 * i] = sha_be32(v.x); w[2 * i + 1] = sha_be32(v.y);
		} else {
			w[i] = sha_be64(v);
		}
	};
	if (o + block <= nbytes) {
		const uint2 *q = reinterpret_cast<const uint2 *>(p + o);
#pragma unroll
		for (int i = 0; i < (int)block / 8; i++) put(i, q[i]);
	} else if (o < nbytes) {
		// the block where the payload ends and the zero extension begins (payload lengths are
		// multiples of 8: the parsers reject anything else)
		const uint64_t rem = nbytes - o;
#pragma unroll
		for (int i = 0; i < (int)block / 8; i++) {
			uint2 v = make_uint2(0u, 0u);
			if (8ull * (uint64_t)i < rem) v = reinterpret_cast<const uint2 *>(p + o)[i];
			put(i, v);
		}
	} else {
#pragma unroll
		for (int i = 0; i < 16; i++) w[i] = 0u;
		if (o >= cover) {
			const uint64_t bits = cover * 8ull;
			w[0] = (W)1 << (8 * sizeof(W) - 1);
			w[15] = (W)bits;      // SHA-512: the 128-bit length, its high word w[14] stays zero
			if constexpr (sizeof(W) == 4) w[14] = (W)(bits >> 32);
		}
	}
}

// The body of k_block_sha256 and k_block_sha512: one thread per record of the (sub-)batch, its key
// compared (block_compare) with the hash H of its bytes, the records compared counted in
// res->*H::counter.  A record whose key is not an H key this stage can check returns at once;
// k_block_check counted it or left it to this kernel.
template <class H>
__device__ __forceinline__ void block_sha(const uint8_t *d_in, const mtz_rec *recs, const uint8_t *d_out,
    const mtz_rec *orecs, uint32_t n, uint32_t mode, uint64_t base, BlockResult *res, const mtz_job *fjobs,
    uint32_t frames)
{
	const uint32_t r = blockIdx.x * H::threads + threadIdx.x;
	if (r >= n) return;
	const mtz_rec rec = recs[r];
	if (rec.type != DRR_WRITE_T) return;
	const uint8_t *hdr = d_in + rec.off;
	block_compare(hdr, rec, r, mode, H::ctype, frames, orecs, d_out, fjobs, res, base, H::counter,
	    [&](const uint8_t *p, uint64_t nbytes, uint64_t cover, int) {
		typename H::word st[8];
#pragma unroll
		for (int i = 0; i < 8; i++) st[i] = H::iv(i);
		const uint64_t nblk = cover / (16 * sizeof(st[0])) + 1ull;
		typename H::word cur[16], nxt[16];
		sha_message_block(p, nbytes, cover, 0, cur);
		for (uint64_t k = 0; k < nblk; k++) {
			if (k + 1ull < nblk) sha_message_block(p, nbytes, cover, k + 1ull, nxt);
			H::compress(st, cur);
#pragma unroll
			for (int i = 0; i < 16; i++) cur[i] = nxt[i];
		}
		const uint64_t *key = reinterpret_cast<const uint64_t *>(hdr + 56);
		bool ok = true;
#pragma unroll
		for (int i = 0; i < 4; i++)
			ok = ok && key[i] == H::key_word(st, i);
		return ok;
	});
}

// block_sha's traits for sha256 keys
#define SHA_THREADS 64
struct Sha256H {
	typedef uint32_t word;
	static constexpr int threads = SHA_THREADS;
	static constexpr uint32_t ctype = ZIO_CKSUM_SHA256;
	static constexpr unsigned long long BlockResult::*counter = &BlockResult::sha256;
	static __device__ __forceinline__ uint32_t iv(int i)      // folds to an immediate for a constant i
	{
		const uint32_t v[8] = { 0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au,
		                        0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u };
		return v[i];
	}
	static __device__ __forceinline__ void compress(uint32_t st[8], uint32_t w[16]) { sha256_compress(st, w); }
	// key word i: the digest's bytes 8i..8i+8 big-endian
	static __device__ __forceinline__ uint64_t key_word(const uint32_t st[8], int i)
	{
		return ((uint64_t)st[2 * i] << 32) | st[2 * i + 1];
	}
};

// The same arguments as k_block_check's but the sums: the hash reads the bytes
__global__ void __launch_bounds__(SHA_THREADS)
k_block_sha256(const uint8_t *__restrict__ d_in, const mtz_rec *__restrict__ recs,
    const uint8_t *__restrict__ d_out, const mtz_rec *__restrict__ orecs, uint32_t n, uint32_t mode,
    uint64_t base, BlockResult *__restrict__ res, const mtz_job *__restrict__ fjobs = nullptr,
    uint32_t frames = 0u)
{
	block_sha<Sha256H>(d_in, recs, d_out, orecs, n, mode, base, res, fjobs, frames);
}

} // namespace mtz
