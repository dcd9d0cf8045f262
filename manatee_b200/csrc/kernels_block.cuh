// kernels_block.cuh -- block-checksum check (MTZ_FLAG_BLOCK_CKSUM): every DRR_WRITE record
// against the on-disk block checksum `zfs send` copies into its header ([EXTERNAL] dmu_send.c
// dump_write(); SURVEY.md App. A.1):
//   byte 48      drr_checksumtype (7 = fletcher4, 8 = sha256: kernels_sha256.cuh,
//                11 = sha512: kernels_sha512.cuh)
//   bytes 56..87 drr_key.ddk_cksum, the block pointer's checksum of the PSIZE bytes on disk
//   bytes 88..95 drr_key.ddk_prop: LSIZE bits 0..15 and PSIZE bits 16..31 as (size/512 - 1),
//                on-disk compression bits 32..38, crypt bit 39
// The stream's own Fletcher-4 chain is re-stamped by every re-encoding mode; this key is not, so it
// ties the bytes a stage hands on to the bytes on the primary's disk.  The check reads only sums K1
// already took (no pass over the stream bytes): the input's body sums start at byte 280, so the
// eight checksum-field words in front of the payload are removed in closed form, and a payload
// shorter than PSIZE is extended by zero words (shift_zeros).
#pragma once
#include "kernels_fletcher.cuh"

namespace mtz {

#define ZIO_CKSUM_FLETCHER4 7u
#define ZIO_CKSUM_SHA256    8u
#define ZIO_CKSUM_SHA512    11u
#define BLK_DC_INHERIT 0u      // "stored raw": the key covers the logical block
#define BLK_DC_OFF     2u
#define BLK_DC_LZ4     15u     // the key covers ZFS's LZ4 frame, zero-padded to PSIZE
#define BLK_DC_LZJB    3u      // ... its lzjb frame (kernels_lzjb.cuh)
#define BLK_DC_ZLE     14u     // ... its zle frame (kernels_lzjb.cuh)
// block_classify's `frames`: the frames VERIFY encodes for the check (kernels_frames.cuh)
#define BLK_FR_LZ4     1u      // MTZ_FLAG_BLOCK_FRAMES: LZ4 frames (K3)
#define BLK_FR_LZJB    2u      // MTZ_FLAG_BLOCK_LZJB: lzjb and zle frames, and in VERIFY and
                               // RECOMPRESS lzjb / zle records that arrive as their disk frame
#define BLK_FR_LOGICAL 4u      // MTZ_FLAG_BLOCK_LOGICAL: the re-encoding modes check keys from the logical
                               // bytes they hold (k_logical_plan, kernels_frames.cuh)
// BlockClass.src: where the bytes a key is compared with are
#define BLK_SRC_IN     0       // the input payload
#define BLK_SRC_OUT    1       // the output payload of a re-encoding mode
#define BLK_SRC_JOB    2       // the check's own job (kernels_frames.cuh): a frame the declared encoder made
                               // for the check, or the logical bytes K2 decoded
#define BLK_SRC_NONE   3       // none: a miss by rule

// The counters carry their mtz_block_stats names.
struct BlockResult {           // device, mirrored to pinned host; zeroed per batch
	unsigned long long logical_ok, frame_ok, frame_miss, skipped;
	unsigned long long sha256;       // records compared by k_block_sha256 (kernels_sha256.cuh)
	unsigned long long sha512;       // records compared by k_block_sha512 (kernels_sha512.cuh)
	unsigned long long frames_encoded;   // LZ4 frames encoded for the check (k_frame_sums, kernels_frames.cuh)
	unsigned long long lzjb_encoded, zle_encoded;   // lzjb / zle frames encoded for the check (likewise)
	unsigned long long logical_checked;    // records compared thanks to MTZ_FLAG_BLOCK_LOGICAL
	unsigned long long first_bad;          // stream index of the first logical mismatch, ~0 none
	unsigned long long first_frame_miss;   // stream index of the first frame mismatch, ~0 none
};
// a batch's results are reset by zeroing everything before first_bad and setting the rest to ~0
static_assert(offsetof(BlockResult, first_frame_miss) == offsetof(BlockResult, first_bad) + 8 &&
    sizeof(BlockResult) == offsetof(BlockResult, first_frame_miss) + 8, "first_bad, first_frame_miss: last");

// zero-state sums of a segment's tail, given the sums of the whole segment and of its 8-word head
// (the inverse of apply(head, tail) for a tail of n words)
__host__ __device__ __forceinline__ Ck4 strip_head8(const Ck4 &whole, const Ck4 &head, uint64_t n)
{
	const uint64_t t2 = tri2(n), t3 = tri3(n);
	Ck4 p;
	p.a = whole.a - head.a;
	p.b = whole.b - head.b - n * head.a;
	p.c = whole.c - head.c - n * head.b - t2 * head.a;
	p.d = whole.d - head.d - n * head.c - t2 * head.b - t3 * head.a;
	return p;
}

// What a record's key lets the stage compare, decided from its header alone, for keys of type
// `ctype`: `what` 0 skipped, 1 the logical block, 2 the disk frame; `src` BLK_SRC_*.
// `have_out` = the output records of a re-encoding mode are at hand; `frames` = BLK_FR_* bits: with
// BLK_FR_LZ4 (VERIFY with MTZ_FLAG_BLOCK_FRAMES) the encoder's LZ4 frames of the raw records are, with
// BLK_FR_LZJB (MTZ_FLAG_BLOCK_LZJB) lzjb and zle keys are checked: against the input payload when
// the record arrives as that frame (VERIFY, RECOMPRESS: passed through), in VERIFY against the
// encoder's frame of a raw record.  With BLK_FR_LOGICAL the re-encoding modes also use the logical
// bytes they hold (the raw input payload, or in DECOMPRESS and RECOMPRESS K2's output for a record that
// arrives LZ4; COMPRESS decodes nothing, so an LZ4 record it is handed stays skipped), rows marked
// `logical`: a raw-on-disk key of an LZ4 record in RECOMPRESS is compared with them; with BLK_FR_LZJB
// an lzjb / zle key with the declared encoder's frame of them, as VERIFY does; and in DECOMPRESS a raw
// record with an LZ4 key is the miss COMPRESS counted for it at the sender (a raw record on the
// lz4-stage-v1 wire is one that stage's encoder stored raw).  Every key type that is checked goes
// through this one table.
struct BlockClass {
	int what, src;
	bool logical;
	uint64_t lsz, psz;
};

__device__ __forceinline__ BlockClass block_classify(const uint8_t *hdr, const mtz_rec &rec, uint32_t mode,
    bool have_out, uint32_t ctype, uint32_t frames = 0u)
{
	const uint64_t prop = *reinterpret_cast<const uint64_t *>(hdr + 88);
	BlockClass c;
	c.lsz = ((prop & 0xffffull) + 1ull) * 512ull;
	c.psz = (((prop >> 16) & 0xffffull) + 1ull) * 512ull;
	c.what = 0; c.src = BLK_SRC_IN; c.logical = false;
	const uint32_t dc = (uint32_t)((prop >> 32) & 0x7full);
	const bool raw_in = rec.comp == 0u, lz4_in = rec.comp == ZIO_LZ4;
	const bool encodes = mode == MTZ_MODE_COMPRESS || mode == MTZ_MODE_RECOMPRESS;
	const bool decodes = mode == MTZ_MODE_DECOMPRESS || mode == MTZ_MODE_RECOMPRESS;
	// the logical bytes of a record that arrives LZ4 exist only where K2 decodes it: not in COMPRESS
	const bool logical = (frames & BLK_FR_LOGICAL) && (raw_in ? (encodes || decodes) : (lz4_in && decodes));
	if (hdr[48] == ctype && prop != 0ull && !((prop >> 39) & 1ull) && c.lsz == rec.lsize) {
		if ((dc == BLK_DC_INHERIT || dc == BLK_DC_OFF) && c.psz == c.lsz) {
			if (raw_in) { c.what = 1; c.src = BLK_SRC_IN; }
			else if (lz4_in && mode == MTZ_MODE_DECOMPRESS && have_out) { c.what = 1; c.src = BLK_SRC_OUT; }
			else if (lz4_in && mode == MTZ_MODE_RECOMPRESS && logical) { c.what = 1; c.src = BLK_SRC_JOB; c.logical = true; }
		} else if (dc == BLK_DC_LZ4) {
			if (lz4_in) { c.what = 2; c.src = BLK_SRC_IN; }
			else if (raw_in && encodes && have_out) { c.what = 2; c.src = BLK_SRC_OUT; }
			else if (raw_in && (frames & BLK_FR_LZ4) && mode == MTZ_MODE_VERIFY) { c.what = 2; c.src = BLK_SRC_JOB; }
			else if (raw_in && mode == MTZ_MODE_DECOMPRESS && logical) { c.what = 2; c.src = BLK_SRC_NONE; c.logical = true; }
		} else if ((frames & BLK_FR_LZJB) && (dc == BLK_DC_LZJB || dc == BLK_DC_ZLE)) {
			if (rec.comp == dc && (mode == MTZ_MODE_VERIFY || mode == MTZ_MODE_RECOMPRESS)) { c.what = 2; c.src = BLK_SRC_IN; }
			else if (raw_in && mode == MTZ_MODE_VERIFY) { c.what = 2; c.src = BLK_SRC_JOB; }
			else if ((raw_in || lz4_in) && logical) { c.what = 2; c.src = BLK_SRC_JOB; c.logical = true; }
		}
	}
	return c;
}

// The verdict of a compared record, `ok` = the bytes match the key.  Record `idx` of the stream.
__device__ __forceinline__ void block_verdict(BlockResult *res, int what, bool ok, uint64_t idx)
{
	if (what == 1) {
		if (ok) atomicAdd(&res->logical_ok, 1ull);
		else atomicMin(&res->first_bad, (unsigned long long)idx);
	} else if (ok) {
		atomicAdd(&res->frame_ok, 1ull);
	} else {
		atomicAdd(&res->frame_miss, 1ull);
		atomicMin(&res->first_frame_miss, (unsigned long long)idx);
	}
}

// The key types checked at all: fletcher4, and type t where `hashed` has bit t set (bit 8:
// k_block_sha256 with MTZ_FLAG_BLOCK_SHA256, bit 11: k_block_sha512 with MTZ_FLAG_BLOCK_SHA512).
__device__ __forceinline__ bool block_key_checked(uint32_t t, uint32_t hashed)
{
	return t == ZIO_CKSUM_FLETCHER4 || (t < 32u && ((hashed >> t) & 1u));
}

// block_classify for the kernels below.  `orecs`: the output records of a re-encoding mode, else
// null.  `have_out` is read only in COMPRESS, DECOMPRESS and RECOMPRESS, where codec_launch_post
// passes the output records together with their sums: `orecs != nullptr` is `osums != nullptr` there.
__device__ __forceinline__ BlockClass block_class(const uint8_t *hdr, const mtz_rec &rec, uint32_t mode,
    uint32_t ctype, uint32_t frames, const mtz_rec *orecs)
{
	return block_classify(hdr, rec, mode, orecs != nullptr, ctype, frames);
}

// Record r's key of type `ctype` against the bytes block_classify picks: the input payload, output
// record r (at `d_out` + its offset) or the check's job r (`fjobs`, kernels_frames.cuh), `nbytes`
// of them at `p`, zero-extended to `cover`.  An encoder storing the block raw where ZFS's
// stored a frame (not that encoder) and bytes longer than the key covers are mismatches;
// `match(p, nbytes, cover, src)` compares the rest.  The verdict goes to `res` as stream record
// `base + r`, after a bump of res->*counter (null: none) and, for a row of MTZ_FLAG_BLOCK_LOGICAL, of
// res->logical_checked.  False: a key this kernel does not check.
template <class Match>
__device__ __forceinline__ bool block_compare(const uint8_t *hdr, const mtz_rec &rec, uint32_t r, uint32_t mode,
    uint32_t ctype, uint32_t frames, const mtz_rec *orecs, const uint8_t *d_out, const mtz_job *fjobs,
    BlockResult *res, uint64_t base, unsigned long long BlockResult::*counter, Match match)
{
	const BlockClass c = block_class(hdr, rec, mode, ctype, frames, orecs);
	if (c.what == 0) return false;
	const uint8_t *p = hdr + DRR_HDR;
	uint64_t nbytes = (uint64_t)rec.payload;
	bool ok = true;
	if (c.src == BLK_SRC_OUT) {
		const mtz_rec o = orecs[r];
		p = d_out + o.off + DRR_HDR;
		nbytes = (uint64_t)o.payload;
		if (c.what == 2 && o.comp != ZIO_LZ4) ok = false;
	} else if (c.src == BLK_SRC_JOB) {
		const mtz_job j = fjobs[r];
		p = reinterpret_cast<const uint8_t *>((uintptr_t)j.dst_off);
		nbytes = (uint64_t)j.out_len;
		if (c.what == 2 && j.out_len >= rec.lsize) ok = false;      // stored raw
	} else if (c.src == BLK_SRC_NONE) {
		ok = false;
	}
	const uint64_t cover = (c.what == 1) ? c.lsz : c.psz;
	if (nbytes > cover) ok = false;
	if (ok) ok = match(p, nbytes, cover, c.src);
	if (counter != nullptr) atomicAdd(&(res->*counter), 1ull);
	if (c.logical) atomicAdd(&res->logical_checked, 1ull);
	block_verdict(res, c.what, ok, base + r);
	return true;
}

// One thread per record.  `isums` are the input's K1 sums (body from byte 280), `orecs`/`osums`
// the output records and their payload sums in the re-encoding modes (null in VERIFY), `d_out` the
// output batch the offsets of `orecs` refer to.  Record r is record `base + r` of the stream.
// `hashed` as block_key_checked's: the keys of those types this stage can check are left to the
// kernel that hashes them instead of being counted as skipped.  `fjobs` / `fsums` (VERIFY with
// MTZ_FLAG_BLOCK_FRAMES or MTZ_FLAG_BLOCK_LZJB, the re-encoding modes with MTZ_FLAG_BLOCK_LOGICAL, else
// null): the check's jobs of kernels_frames.cuh and the sums of their bytes.  `frames`:
// block_classify's BLK_FR_* bits.
#define BLK_THREADS 128
__global__ void __launch_bounds__(BLK_THREADS)
k_block_check(const uint8_t *__restrict__ d_in, const mtz_rec *__restrict__ recs,
    const RecSums *__restrict__ isums, const mtz_rec *__restrict__ orecs,
    const RecSums *__restrict__ osums, const uint8_t *__restrict__ d_out, uint32_t n, uint32_t mode,
    uint64_t base, BlockResult *__restrict__ res, uint32_t hashed, const mtz_job *__restrict__ fjobs = nullptr,
    const RecSums *__restrict__ fsums = nullptr, uint32_t frames = 0u)
{
	const uint32_t r = blockIdx.x * BLK_THREADS + threadIdx.x;
	if (r >= n) return;
	const mtz_rec rec = recs[r];
	if (rec.type != DRR_WRITE_T) return;
	const uint8_t *hdr = d_in + rec.off;
	const bool checked = block_compare(hdr, rec, r, mode, ZIO_CKSUM_FLETCHER4, frames, orecs, d_out, fjobs, res,
	    base, nullptr, [&](const uint8_t *, uint64_t nbytes, uint64_t cover, int src) {
		Ck4 sums;
		if (src == BLK_SRC_IN) {
			const RecSums s = isums[r];
			const Ck4 zero = { 0, 0, 0, 0 };
			sums = strip_head8(s.body, fold_cksum_words(zero, s.emb), s.nbody - 8u);
		} else {
			sums = (src == BLK_SRC_OUT ? osums : fsums)[r].body;
		}
		return ck_eq(shift_zeros(sums, (cover - nbytes) >> 2), load_ck(hdr + 56));
	});
	if (!checked) {
		const uint32_t t = hdr[48];
		if (!block_key_checked(t, hashed) || block_class(hdr, rec, mode, t, frames, orecs).what == 0)
			atomicAdd(&res->skipped, 1ull);
	}
}

} // namespace mtz
