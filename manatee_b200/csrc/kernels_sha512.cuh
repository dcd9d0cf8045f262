// kernels_sha512.cuh -- block checksums with SHA-512 keys (MTZ_FLAG_BLOCK_SHA512): the records
// k_block_check leaves alone because their drr_checksumtype is 11 ([EXTERNAL] ZIO_CHECKSUM_SHA512,
// checksum=sha512).  Same table (block_classify), same bytes, same zero extension to the covered
// size, same verdicts as fletcher4 and sha256 keys; only the hash differs.
//
// Key format ([EXTERNAL] OpenZFS abd_checksum_sha512_native; validated only against the FIPS 180-4
// known answers, no real checksum=sha512 stream has been through it): the hash is SHA-512/256 (the
// SHA-512 compression from the SHA-512/256 initial value, truncated to 256 bits), and the 32 digest
// bytes are the key bytes in order -- unlike sha256 keys there is no BE_64 per word.  The words travel
// in the stream as native little-endian u64, so word i = bswap64(H[i]) with H the first four state
// words of the final hash.  The message is a multiple of 512 bytes: its padding is always one extra
// 128-byte block, and the high word of the 128-bit length is zero.
//
// One thread per record as for sha256 (the hash is serial within a message).  Every 64-bit operation
// runs on the 32-bit ALU: rotations are two funnel shifts on the halves, additions carry pairs.  The
// round loop is unrolled (the 80 constants fold into immediates), the message schedule is a rolling
// 16-word window in registers, and the next 128-byte block is loaded while the current one compresses.
#pragma once
#include "kernels_sha256.cuh"

namespace mtz {

// round constant t; called with a constant t in the unrolled round loop, so it folds to an immediate
__device__ __forceinline__ uint64_t sha512_k(int t)
{
	const uint64_t k[80] = {
		0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull,
		0x3956c25bf348b538ull, 0x59f111f1b605d019ull, 0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull,
		0xd807aa98a3030242ull, 0x12835b0145706fbeull, 0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull,
		0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull, 0xc19bf174cf692694ull,
		0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull, 0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull,
		0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull,
		0x983e5152ee66dfabull, 0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull,
		0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull, 0x06ca6351e003826full, 0x142929670a0e6e70ull,
		0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull, 0x53380d139d95b3dfull,
		0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull,
		0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull, 0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull,
		0xd192e819d6ef5218ull, 0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull,
		0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull, 0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull,
		0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull, 0x5b9cca4f7763e373ull, 0x682e6ff3d6b2b8a3ull,
		0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull,
		0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull,
		0xca273eceea26619cull, 0xd186b8c721c0c207ull, 0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull,
		0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull, 0x113f9804bef90daeull, 0x1b710b35131c471bull,
		0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull, 0x431d67c49c100d4cull,
		0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull, 0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull,
	};
	return k[t];
}

// 64-bit rotate right by a constant n (1..63) as two 32-bit funnel shifts on the halves
__device__ __forceinline__ uint64_t sha_rotr64(uint64_t x, int n)
{
	const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
	if (n < 32) return sha_join(__funnelshift_r(lo, hi, n), __funnelshift_r(hi, lo, n));
	return sha_join(__funnelshift_r(hi, lo, n - 32), __funnelshift_r(lo, hi, n - 32));
}

// FIPS 180-4 SHA-512 compression of one 128-byte block (`w` = its 16 big-endian words, consumed)
__device__ __forceinline__ void sha512_compress(uint64_t st[8], uint64_t w[16])
{
	uint64_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
	for (int t = 0; t < 80; t++) {
		if (t >= 16) {
			const uint64_t x = w[(t - 15) & 15], y = w[(t - 2) & 15];
			const uint64_t s0 = sha_rotr64(x, 1) ^ sha_rotr64(x, 8) ^ (x >> 7);
			const uint64_t s1 = sha_rotr64(y, 19) ^ sha_rotr64(y, 61) ^ (y >> 6);
			w[t & 15] += s0 + w[(t - 7) & 15] + s1;
		}
		const uint64_t t1 = h + (sha_rotr64(e, 14) ^ sha_rotr64(e, 18) ^ sha_rotr64(e, 41)) +
		    ((e & f) ^ (~e & g)) + sha512_k(t) + w[t & 15];
		const uint64_t t2 = (sha_rotr64(a, 28) ^ sha_rotr64(a, 34) ^ sha_rotr64(a, 39)) +
		    ((a & b) ^ (a & c) ^ (b & c));
		h = g; g = f; f = e; e = d + t1;
		d = c; c = b; b = a; a = t1 + t2;
	}
	st[0] += a; st[1] += b; st[2] += c; st[3] += d;
	st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// block_sha's traits for sha512 keys
#define SHA512_THREADS 64
struct Sha512H {
	typedef uint64_t word;
	static constexpr int threads = SHA512_THREADS;
	static constexpr uint32_t ctype = ZIO_CKSUM_SHA512;
	static constexpr unsigned long long BlockResult::*counter = &BlockResult::sha512;
	// SHA-512/256 initial hash value (FIPS 180-4 5.3.6.2)
	static __device__ __forceinline__ uint64_t iv(int i)      // folds to an immediate for a constant i
	{
		const uint64_t v[8] = { 0x22312194fc2bf72cull, 0x9f555fa3c84c64c2ull, 0x2393b86b6f53b151ull,
		                        0x963877195940eabdull, 0x96283ee2a88effe3ull, 0xbe5e1e2553863992ull,
		                        0x2b0199fc2c85b8aaull, 0x0eb72ddc81c52ca2ull };
		return v[i];
	}
	static __device__ __forceinline__ void compress(uint64_t st[8], uint64_t w[16]) { sha512_compress(st, w); }
	// key word i: the digest's bytes 8i..8i+8 in order
	static __device__ __forceinline__ uint64_t key_word(const uint64_t st[8], int i)
	{
		return sha_be64(make_uint2((uint32_t)st[i], (uint32_t)(st[i] >> 32)));
	}
};

// The same arguments as k_block_sha256's
__global__ void __launch_bounds__(SHA512_THREADS)
k_block_sha512(const uint8_t *__restrict__ d_in, const mtz_rec *__restrict__ recs,
    const uint8_t *__restrict__ d_out, const mtz_rec *__restrict__ orecs, uint32_t n, uint32_t mode,
    uint64_t base, BlockResult *__restrict__ res, const mtz_job *__restrict__ fjobs = nullptr,
    uint32_t frames = 0u)
{
	block_sha<Sha512H>(d_in, recs, d_out, orecs, n, mode, base, res, fjobs, frames);
}

} // namespace mtz
