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

// Block k of the message "nbytes of `p`, zeros up to `cover`, FIPS 180-4 padding" as 16 big-endian
// words.  `p` is 8-byte aligned, `nbytes` a multiple of 8; no byte at or past p[nbytes] is read (the
// zeros are arithmetic).
__device__ __forceinline__ void sha256_message_block(const uint8_t *__restrict__ p, uint64_t nbytes,
    uint64_t cover, uint64_t k, uint32_t w[16])
{
	const uint64_t o = k * 64ull;
	if (o + 64ull <= nbytes) {
		const uint2 *q = reinterpret_cast<const uint2 *>(p + o);
#pragma unroll
		for (int i = 0; i < 8; i++) {
			const uint2 v = q[i];
			w[2 * i] = sha_be32(v.x); w[2 * i + 1] = sha_be32(v.y);
		}
	} else if (o < nbytes) {
		// the block where the payload ends and the zero extension begins (payload lengths are
		// multiples of 8: the parsers reject anything else)
		const uint64_t rem = nbytes - o;
#pragma unroll
		for (int i = 0; i < 8; i++) {
			uint2 v = make_uint2(0u, 0u);
			if (8ull * (uint64_t)i < rem) v = reinterpret_cast<const uint2 *>(p + o)[i];
			w[2 * i] = sha_be32(v.x); w[2 * i + 1] = sha_be32(v.y);
		}
	} else {
#pragma unroll
		for (int i = 0; i < 16; i++) w[i] = 0u;
		if (o >= cover) {
			const uint64_t bits = cover * 8ull;
			w[0] = 0x80000000u;
			w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits;
		}
	}
}

// One thread per record of the (sub-)batch, the same arguments as k_block_check plus the output
// batch base (`orecs[r].off` is relative to `d_out`).  A record whose key is not a sha256 key this
// stage can check returns at once; k_block_check counted it or left it to this kernel.
#define SHA_THREADS 64
__global__ void __launch_bounds__(SHA_THREADS)
k_block_sha256(const uint8_t *__restrict__ d_in, const mtz_rec *__restrict__ recs,
    const uint8_t *__restrict__ d_out, const mtz_rec *__restrict__ orecs, uint32_t n, uint32_t mode,
    uint64_t base, BlockResult *__restrict__ res, const mtz_job *__restrict__ fjobs = nullptr,
    uint32_t frames = 0u)
{
	const uint32_t r = blockIdx.x * SHA_THREADS + threadIdx.x;
	if (r >= n) return;
	const mtz_rec rec = recs[r];
	if (rec.type != DRR_WRITE_T) return;
	const uint8_t *hdr = d_in + rec.off;
	const BlockClass c = block_classify(hdr, rec, mode, orecs != nullptr, ZIO_CKSUM_SHA256, frames);
	if (c.what == 0) return;
	const uint8_t *p;
	uint64_t nbytes;
	bool ok = true;
	if (c.src == 0) {
		p = hdr + DRR_HDR;
		nbytes = (uint64_t)rec.payload;
	} else if (fjobs == nullptr) {
		const mtz_rec o = orecs[r];
		p = d_out + o.off + DRR_HDR;
		nbytes = (uint64_t)o.payload;
		// the stage's encoder stored the block raw where ZFS's stored a frame: not that encoder
		if (c.what == 2 && o.comp != ZIO_LZ4) ok = false;
	} else {
		// VERIFY with MTZ_FLAG_BLOCK_FRAMES / _LZJB: the declared encoder's frame (kernels_frames.cuh)
		const mtz_job j = fjobs[r];
		p = reinterpret_cast<const uint8_t *>((uintptr_t)j.dst_off);
		nbytes = (uint64_t)j.out_len;
		if (j.out_len >= rec.lsize) ok = false;
	}
	const uint64_t cover = (c.what == 1) ? c.lsz : c.psz;
	if (nbytes > cover) ok = false;
	if (ok) {
		uint32_t st[8] = { 0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au,
		                   0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u };
		const uint64_t nblk = cover / 64ull + 1ull;
		uint32_t cur[16], nxt[16];
		sha256_message_block(p, nbytes, cover, 0, cur);
		for (uint64_t k = 0; k < nblk; k++) {
			if (k + 1ull < nblk) sha256_message_block(p, nbytes, cover, k + 1ull, nxt);
			sha256_compress(st, cur);
#pragma unroll
			for (int i = 0; i < 16; i++) cur[i] = nxt[i];
		}
		const uint64_t *key = reinterpret_cast<const uint64_t *>(hdr + 56);
#pragma unroll
		for (int i = 0; i < 4; i++)
			ok = ok && key[i] == (((uint64_t)st[2 * i] << 32) | st[2 * i + 1]);
	}
	atomicAdd(&res->sha256, 1ull);
	block_verdict(res, c.what, ok, base + r);
}

} // namespace mtz
