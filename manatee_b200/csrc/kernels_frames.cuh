// kernels_frames.cuh -- the frames of the block check in VERIFY (MTZ_FLAG_BLOCK_FRAMES,
// MTZ_FLAG_BLOCK_LZJB).  A block ZFS stored compressed has a key over its disk frame, zero-padded to
// PSIZE; a VERIFY stage that receives the block raw (`zfs send` without -c) has no frame to compare.
// With the flags it makes one with the declared encoder into a scratch beside the batch, and the
// checks compare that frame by the rules of COMPRESS, which compares its own encoder output: the
// stage hands on the input bytes untouched either way.
//   k_frame_plan  one job per record: the raw records whose key covers an LZ4 (MTZ_FLAG_BLOCK_FRAMES),
//                 lzjb or zle frame (MTZ_FLAG_BLOCK_LZJB), the decision block_classify's and the codec
//                 in the job's src_len; an empty job for every other record
//   K3            k3_lz4_encode over the LZ4 jobs: out_len = PSIZE of the frame, or lsize = stored raw
//   k_lzjb_encode, k_zle_encode (kernels_lzjb.cuh): likewise over the lzjb and zle jobs
//   k_frame_sums  Fletcher-4 sums of each frame, one warp per record (warp_fletcher rows)
// k_block_check, k_block_sha256 and k_block_sha512 then read the frame through the jobs.
#pragma once
#include "kernels_block.cuh"
#include "kernels_lzjb.cuh"

namespace mtz {

// Record r's slot is scratch + (rec.off & ~15) - base_off: its frame is at most lsize bytes and the
// record itself spans 312 + lsize bytes of the batch, so the slots of a batch do not overlap and
// the scratch needs no more bytes than the batch (base_off 16-aligned, at or before the first
// header).  `hashed` as block_key_checked's; `frames`: block_classify's BLK_FR_* bits.  A job's
// src_len is its codec (BLK_DC_LZ4 / _LZJB / _ZLE).
// `k3_skip` (null unless both flags are on): 1 for each job K3 must leave to the other encoders.
#define FRP_THREADS 128
__global__ void __launch_bounds__(FRP_THREADS)
k_frame_plan(const uint8_t *__restrict__ d_in, const mtz_rec *__restrict__ recs, uint32_t n,
    uint32_t hashed, uint64_t base_off, uint8_t *scratch, mtz_job *__restrict__ jobs, uint32_t frames,
    uint32_t *__restrict__ k3_skip)
{
	const uint32_t r = blockIdx.x * FRP_THREADS + threadIdx.x;
	if (r >= n) return;
	const mtz_rec rec = recs[r];
	mtz_job j;
	j.src_off = j.dst_off = 0; j.src_len = 0; j.lsize = 0; j.out_len = 0; j.status = 0;
	if (rec.type == DRR_WRITE_T) {
		const uint8_t *hdr = d_in + rec.off;
		const uint32_t t = hdr[48];
		if (block_key_checked(t, hashed)) {
			const BlockClass c = block_classify(hdr, rec, MTZ_MODE_VERIFY, false, t, frames);
			if (c.what == 2 && c.src == 1) {
				j.src_len = (uint32_t)((*reinterpret_cast<const uint64_t *>(hdr + 88) >> 32) & 0x7full);
				j.src_off = (uint64_t)(uintptr_t)(hdr + DRR_HDR);
				j.dst_off = (uint64_t)(uintptr_t)(scratch + ((rec.off & ~15ull) - base_off));
				j.lsize = rec.lsize;
			}
		}
	}
	jobs[r] = j;
	if (k3_skip != nullptr) k3_skip[r] = j.src_len != BLK_DC_LZ4;
}

// One warp per record (grid-stride): zero-state sums of the frame its encoder left at jobs[r].dst_off
// into sums[r].body, and the record counted in res->frames_encoded, lzjb_encoded or zle_encoded by its
// codec.  A frame the encoder stored raw (out_len == lsize) has no sums: the checks count it as a
// miss without reading them.
__global__ void __launch_bounds__(K1_THREADS)
k_frame_sums(const mtz_job *__restrict__ jobs, uint32_t n, RecSums *__restrict__ sums,
    BlockResult *__restrict__ res)
{
	const int lane = threadIdx.x & 31;
	const uint32_t gw = blockIdx.x * K1_WARPS + (threadIdx.x >> 5);
	const uint32_t nw = gridDim.x * K1_WARPS;
	for (uint32_t r = gw; r < n; r += nw) {
		const mtz_job j = jobs[r];
		if (j.lsize == 0u) continue;
		Ck4 acc = { 0, 0, 0, 0 };
		if (j.out_len < j.lsize) {
			// frames are whole 512-byte sectors in a 16-aligned slot: every chunk is whole rows
			const uint8_t *p = reinterpret_cast<const uint8_t *>((uintptr_t)j.dst_off);
			const uint32_t nwords = j.out_len >> 2;
			for (uint32_t w0 = 0; w0 < nwords;) {
				const uint32_t w1 = min(nwords, w0 + MTZ_K1_MAX_ROWS * 128u);
				Ck4 q = warp_fletcher(p + 4ull * w0, w1 - w0, lane);
				if (w1 != nwords) q = shift_zeros(q, (uint64_t)(nwords - w1));
				acc.a += q.a; acc.b += q.b; acc.c += q.c; acc.d += q.d;
				w0 = w1;
			}
		}
		if (lane == 0) {
			sums[r].body = acc;
			atomicAdd(j.src_len == BLK_DC_LZJB ? &res->lzjb_encoded : j.src_len == BLK_DC_ZLE ? &res->zle_encoded :
			    &res->frames_encoded, 1ull);
		}
	}
}

} // namespace mtz
