/*
 * lz4hc_ref.c -- the high-ratio LZ4 encoder of MTZ_FLAG_LZ4_HC, restated serially on the CPU.
 * Test infrastructure: tests/lz4hc_ref.py compiles it (with oracle/stream.c for the stream walk)
 * and the kernel k3h_lz4hc_encode (manatee_b200/csrc/kernels_lz4hc.cuh) must equal it byte for byte.
 *
 * The parse (DESIGN.md section 1, "COMPRESS with MTZ_FLAG_LZ4_HC"):
 *   hash(p) = (LE32(src+p) * 2654435761 mod 2^32) >> 20, 4096 buckets of the last 16 positions
 *   inserted with that hash (the oldest is dropped from a full bucket), empty at the start of a block.
 *   Every position below p is inserted before p is searched.  The candidates at p < n-12 are the
 *   bucket's entries c with p-c <= 65535 and LE32(src+c) == LE32(src+p); each is compared for at most
 *   min(64, n-5-p) bytes, the longest wins (the larger c on a tie), and only the winner is extended
 *   up to n-5.  Greedy: no lazy step, no backward extension.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define HC_MINMATCH 4
#define HC_MFLIMIT 12
#define HC_LASTLITERALS 5
#define HC_MAXOFF 65535u
#define HC_HB 12
#define HC_W 16
#define HC_CAP 64

static uint32_t
le32(const uint8_t *p)
{
	return ((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24));
}

static uint32_t
hc_hash(const uint8_t *p)
{
	return ((le32(p) * 2654435761u) >> (32 - HC_HB));
}

/* appends one length extension (v = len - 15) at dst[op]; returns the new op or -1 past cap */
static long
put_ext(uint8_t *dst, long op, long cap, uint32_t v)
{
	for (; v >= 255u; v -= 255u) {
		if (op >= cap) return (-1);
		dst[op++] = 255;
	}
	if (op >= cap) return (-1);
	dst[op++] = (uint8_t)v;
	return (op);
}

/* one sequence: literals src[anchor, anchor+lit), then (off, ml) unless ml == 0 */
static long
put_seq(uint8_t *dst, long op, long cap, const uint8_t *lits, uint32_t lit, uint32_t off, uint32_t ml)
{
	uint32_t mcode = ml ? ml - HC_MINMATCH : 0;
	if (op >= cap) return (-1);
	dst[op++] = (uint8_t)(((lit >= 15 ? 15 : lit) << 4) | (mcode >= 15 ? 15 : mcode));
	if (lit >= 15 && (op = put_ext(dst, op, cap, lit - 15)) < 0) return (-1);
	if ((long)lit > cap - op) return (-1);
	memcpy(dst + op, lits, lit);
	op += lit;
	if (ml == 0) return (op);
	if (cap - op < 2) return (-1);
	dst[op++] = (uint8_t)off;
	dst[op++] = (uint8_t)(off >> 8);
	if (mcode >= 15 && (op = put_ext(dst, op, cap, mcode - 15)) < 0) return (-1);
	return (op);
}

/* raw LZ4 block of src[0, n) into dst[0, cap); returns its length, 0 if it does not fit */
int
orc_lz4hc_compress_block(const uint8_t *src, int n, uint8_t *dst, int cap)
{
	uint32_t *tab, *cnt;
	long op = 0, mflimit = (long)n - HC_MFLIMIT, matchlimit = (long)n - HC_LASTLITERALS;
	long p = 0, anchor = 0, ins = 0;

	if (n < 0 || cap < 0) return (0);
	tab = (uint32_t *)malloc(sizeof (uint32_t) * (HC_W << HC_HB));
	cnt = (uint32_t *)calloc(1u << HC_HB, sizeof (uint32_t));
	if (tab == NULL || cnt == NULL) { free(tab); free(cnt); return (0); }

	while (p < mflimit) {
		const uint32_t h = hc_hash(src + p), v = le32(src + p);
		const long lim = (matchlimit - p) < HC_CAP ? (matchlimit - p) : HC_CAP;
		long best = 0, bc = -1, ml;
		uint32_t i, k;

		for (; ins < p; ins++) {                     /* every position below p is in the table */
			const uint32_t hi = hc_hash(src + ins);
			tab[hi * HC_W + (cnt[hi] % HC_W)] = (uint32_t)ins;
			cnt[hi]++;
		}
		k = cnt[h] < HC_W ? cnt[h] : HC_W;
		for (i = 0; i < k; i++) {
			const long c = tab[h * HC_W + ((cnt[h] - 1 - i) % HC_W)];
			long len = 0;
			if ((unsigned long)(p - c) > HC_MAXOFF || le32(src + c) != v) continue;
			while (len < lim && src[c + len] == src[p + len]) len++;
			if (len > best || (len == best && c > bc)) { best = len; bc = c; }
		}
		if (bc < 0) { p++; continue; }
		ml = best;
		if (ml == HC_CAP)
			while (p + ml < matchlimit && src[bc + ml] == src[p + ml]) ml++;
		op = put_seq(dst, op, cap, src + anchor, (uint32_t)(p - anchor), (uint32_t)(p - bc), (uint32_t)ml);
		if (op < 0) break;
		p += ml;
		anchor = p;
	}
	free(tab);
	free(cnt);
	if (op < 0) return (0);
	op = put_seq(dst, op, cap, src + anchor, (uint32_t)(n - anchor), 0, 0);
	return (op < 0 ? 0 : (int)op);
}

/* zio_compress_data + sector rounding with this encoder (the rule of orc_zfs_lz4_compress): returns
 * psize and fills dst[0, psize) with BE32 clen | block | zero pad, or lsize when the block is stored raw */
size_t
orc_zfs_lz4hc_compress(const uint8_t *src, size_t lsize, uint8_t *dst)
{
	size_t d_len = lsize - lsize / 8, psize;
	int clen;

	if (lsize < 1024 || lsize > (16u << 20) || d_len < 4) return (lsize);
	clen = orc_lz4hc_compress_block(src, (int)lsize, dst + 4, (int)(d_len - 4));
	if (clen <= 0 || 4 + (size_t)clen > d_len) return (lsize);
	psize = (4 + (size_t)clen + 511) & ~(size_t)511;
	if (psize >= lsize) return (lsize);
	dst[0] = (uint8_t)(clen >> 24); dst[1] = (uint8_t)(clen >> 16);
	dst[2] = (uint8_t)(clen >> 8);  dst[3] = (uint8_t)clen;
	memset(dst + 4 + clen, 0, psize - 4 - (size_t)clen);
	return (psize);
}
