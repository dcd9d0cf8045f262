/* lzjb_zfs.c -- TEST INFRASTRUCTURE: ZFS's lzjb and zle encoders and decoders, restated in C
 * ([EXTERNAL] lzjb.c, zle.c), driven the way zio_compress_data drives them.  Built and loaded by
 * tests/block_lzjb_ref.py (compiled into a temporary directory on first use); the GPU encoders of
 * manatee_b200/csrc/kernels_lzjb.cuh are held to it.
 *
 * lzjb's table keeps the low 16 bits of source POINTERS, so its output depends on the address of
 * the source buffer modulo 1024 (its "phase"): zfs_lzjb_compress copies the block to that phase of a
 * 1 KiB-aligned buffer and runs the encoder on the real pointers. */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef unsigned char uchar_t;
#define NBBY 8

#define MATCH_BITS  6
#define MATCH_MIN   3
#define MATCH_MAX   ((1 << MATCH_BITS) + (MATCH_MIN - 1))
#define OFFSET_MASK ((1 << (16 - MATCH_BITS)) - 1)
#define LEMPEL_SIZE 1024

static size_t lzjb_compress(void *s_start, void *d_start, size_t s_len, size_t d_len)
{
	uchar_t *src = s_start;
	uchar_t *dst = d_start;
	uchar_t *cpy;
	uchar_t *copymap = NULL;
	int copymask = 1 << (NBBY - 1);
	int mlen, offset, hash;
	uint16_t *hp;
	uint16_t lempel[LEMPEL_SIZE] = { 0 };

	while (src < (uchar_t *)s_start + s_len) {
		if ((copymask <<= 1) == (1 << NBBY)) {
			if (dst >= (uchar_t *)d_start + d_len - 1 - 2 * NBBY)
				return s_len;
			copymask = 1;
			copymap = dst;
			*dst++ = 0;
		}
		if (src > (uchar_t *)s_start + s_len - MATCH_MAX) {
			*dst++ = *src++;
			continue;
		}
		hash = (src[0] << 16) + (src[1] << 8) + src[2];
		hash += hash >> 9;
		hash += hash >> 5;
		hp = &lempel[hash & (LEMPEL_SIZE - 1)];
		offset = (intptr_t)(src - *hp) & OFFSET_MASK;
		*hp = (uint16_t)(uintptr_t)src;
		cpy = src - offset;
		if (cpy >= (uchar_t *)s_start && cpy != src &&
		    src[0] == cpy[0] && src[1] == cpy[1] && src[2] == cpy[2]) {
			*copymap |= copymask;
			for (mlen = MATCH_MIN; mlen < MATCH_MAX; mlen++)
				if (src[mlen] != cpy[mlen])
					break;
			*dst++ = ((mlen - MATCH_MIN) << (NBBY - MATCH_BITS)) | (offset >> NBBY);
			*dst++ = (uchar_t)offset;
			src += mlen;
		} else {
			*dst++ = *src++;
		}
	}
	return dst - (uchar_t *)d_start;
}

static int lzjb_decompress(void *s_start, void *d_start, size_t s_len, size_t d_len)
{
	uchar_t *src = s_start;
	uchar_t *s_end = src + s_len;
	uchar_t *dst = d_start;
	uchar_t *d_end = (uchar_t *)d_start + d_len;
	uchar_t *cpy;
	uchar_t copymap = 0;
	int copymask = 1 << (NBBY - 1);

	while (dst < d_end) {
		if ((copymask <<= 1) == (1 << NBBY)) {
			if (src >= s_end)
				return -1;
			copymask = 1;
			copymap = *src++;
		}
		if (copymap & copymask) {
			if (src + 2 > s_end)
				return -1;
			int mlen = (src[0] >> (NBBY - MATCH_BITS)) + MATCH_MIN;
			int offset = ((src[0] << NBBY) | src[1]) & OFFSET_MASK;
			src += 2;
			if ((cpy = dst - offset) < (uchar_t *)d_start)
				return -1;
			if (mlen > (d_end - dst))
				mlen = d_end - dst;
			while (--mlen >= 0)
				*dst++ = *cpy++;
		} else {
			if (src >= s_end)
				return -1;
			*dst++ = *src++;
		}
	}
	return 0;
}

static size_t zle_compress(void *s_start, void *d_start, size_t s_len, size_t d_len, int n)
{
	uchar_t *src = s_start;
	uchar_t *dst = d_start;
	uchar_t *s_end = src + s_len;
	uchar_t *d_end = dst + d_len;

	while (src < s_end && dst < d_end - 1) {
		uchar_t *first = src;
		uchar_t *len = dst++;
		if (src[0] == 0) {
			uchar_t *last = src + (256 - n);
			while (src < (last < s_end ? last : s_end) && src[0] == 0)
				src++;
			*len = src - first - 1 + n;
		} else {
			uchar_t *last = src + n;
			if (d_end - dst < n)
				break;
			while (src < (last < s_end ? last : s_end) - 1 && (src[0] | src[1]))
				*dst++ = *src++;
			if (src[0])
				*dst++ = *src++;
			*len = src - first - 1;
		}
	}
	return src == s_end ? (size_t)(dst - (uchar_t *)d_start) : s_len;
}

static int zle_decompress(void *s_start, void *d_start, size_t s_len, size_t d_len, int n)
{
	uchar_t *src = s_start;
	uchar_t *dst = d_start;
	uchar_t *s_end = src + s_len;
	uchar_t *d_end = dst + d_len;

	while (src < s_end && dst < d_end) {
		int len = 1 + *src++;
		if (len <= n) {
			if (src + len > s_end || dst + len > d_end)
				return -1;
			while (len-- != 0)
				*dst++ = *src++;
		} else {
			len -= n;
			if (dst + len > d_end)
				return -1;
			while (len-- != 0)
				*dst++ = 0;
		}
	}
	return dst == d_end ? 0 : -1;
}

/* zio_compress_data's rule: d_len = s_len - s_len/8; a result above d_len is "stored raw";
 * otherwise the frame is zero-padded to a whole 512-byte sector and a pad that reaches s_len is
 * "stored raw" too.  Returns the PSIZE of the frame written to dst (s_len bytes of room), or s_len
 * when the block is stored raw; *c_len gets the encoder's own result. */
static size_t zio_rule(uchar_t *dst, size_t c_len, size_t s_len)
{
	size_t d_len = s_len - (s_len >> 3);
	if (c_len > d_len)
		return s_len;
	size_t ps = (c_len + 511) & ~(size_t)511;
	if (ps >= s_len)
		return s_len;
	memset(dst + c_len, 0, ps - c_len);
	return ps;
}

size_t orc_zfs_lzjb_compress(const void *src, size_t s_len, void *dst, size_t *c_len, unsigned phase)
{
	uchar_t *buf = aligned_alloc(1024, ((s_len + 1024 + 1023) / 1024) * 1024);
	if (buf == NULL)
		return 0;
	memcpy(buf + (phase & 1023), src, s_len);
	*c_len = lzjb_compress(buf + (phase & 1023), dst, s_len, s_len - (s_len >> 3));
	free(buf);
	return zio_rule(dst, *c_len, s_len);
}

size_t orc_zfs_zle_compress(const void *src, size_t s_len, void *dst, size_t *c_len)
{
	*c_len = zle_compress((void *)src, dst, s_len, s_len - (s_len >> 3), 64);
	return zio_rule(dst, *c_len, s_len);
}

int orc_lzjb_decompress(const void *src, size_t s_len, void *dst, size_t d_len)
{
	return lzjb_decompress((void *)src, dst, s_len, d_len);
}

int orc_zle_decompress(const void *src, size_t s_len, void *dst, size_t d_len)
{
	return zle_decompress((void *)src, dst, s_len, d_len, 64);
}
