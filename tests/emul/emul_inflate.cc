// emul_inflate.cc -- TEST INFRASTRUCTURE: k_inflate of COMPRESS with MTZ_FLAG_GZIP_IN
// (manatee_b200/csrc/kernels_inflate.cuh) launched as the pipeline launches it, on the SIMT emulator
// (tests/emul/cuda_runtime.h), one job per call.  Built on its own (with warp_emul.cc); the guard-page
// buffers come from emul_kernels.cc's build.
#include "cuda_runtime.h"
#include "../../manatee_b200/csrc/kernels_codec.cuh"
#include "../../manatee_b200/csrc/kernels_inflate.cuh"

extern "C" {

// the zlib stream [src, src + s_len) of a record with drr_compressiontype `comp` inflated to lsize bytes
// at dst by k_inflate in a grid of `grid` CTAs whose job is number `slot` of `njobs` (the others empty):
// MTZ_OK or MTZ_ECODEC; -100 a job other than the record's was touched, 77 the job was left alone
int32_t emu_inflate(uint32_t comp, const uint8_t *src, uint32_t s_len, uint8_t *dst, uint32_t lsize,
    uint32_t slot, uint32_t njobs, uint32_t grid)
{
	using namespace mtz;
	mtz_rec recs[64];
	mtz_job jobs[64];
	if (njobs > 64 || slot >= njobs) return -101;
	for (uint32_t i = 0; i < njobs; i++) {
		memset(&recs[i], 0, sizeof recs[i]);
		memset(&jobs[i], 0, sizeof jobs[i]);
		recs[i].type = 3; recs[i].comp = comp; jobs[i].status = 77;
	}
	jobs[slot].src_off = (uint64_t)(uintptr_t)src; jobs[slot].dst_off = (uint64_t)(uintptr_t)dst;
	jobs[slot].src_len = s_len; jobs[slot].lsize = lsize;
	emu::launch(grid, INFL_THREADS, [&] { k_inflate(recs, jobs, njobs); });
	for (uint32_t i = 0; i < njobs; i++)
		if (i != slot && (jobs[i].status != 77 || jobs[i].out_len != 0)) return -100;
	if (jobs[slot].status == MTZ_OK && jobs[slot].out_len != lsize) return -102;
	return jobs[slot].status;
}

} // extern "C"
