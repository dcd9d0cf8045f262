// kernels_codec.cuh -- K4: the re-encoding pipeline around K2/K3 for the stage
// modes COMPRESS / DECOMPRESS / RECOMPRESS (include/manatee_gpu.h):
//   plan     classify records, lay out decode/encode scratch, fill K2/K3 jobs
//   layout   per-record output length -> output offsets (exclusive scan)
//   assemble copy header (compressiontype / compressed_size / BEGIN flags
//            rewritten) + payload from its source into the output slice
//   stamp    dump_record() checksum chain over the OUTPUT records
// Stream semantics: illumos dmu_send.c dump_record() ([EXTERNAL], SURVEY.md
// App. A.1-A.2); transform definitions: oracle/stream.c walk().  The reference
// itself only pipes bytes (lib/backupSender.js:179, lib/zfsClient.js:826).
#pragma once
#include "kernels_fletcher.cuh"
#include "kernels_lz4.cuh"

namespace mtz {

#define CF_DEC    1u      // payload is a frame that this mode decodes: ZFS-LZ4 (K2), or in COMPRESS with
                          // MTZ_FLAG_COMPRESSED_IN lzjb / zle (k_lzjb_decode / k_zle_decode) and with
                          // MTZ_FLAG_GZIP_IN gzip-1 .. gzip-9 (k_inflate); in DECOMPRESS with
                          // MTZ_FLAG_GZIP_WIRE also gzip-1 .. gzip-9 (k_inflate over the second job table)
#define CF_ENC    2u      // (decoded or raw) logical payload is offered to the encoder
#define CF_WRITE  4u
#define CF_PASS   8u      // COMPRESS with MTZ_FLAG_COMPRESSED_IN: an LZ4 frame, and with MTZ_FLAG_GZIP_WIRE
                          // a gzip frame, forwarded as it is
#define CF_BAD    16u     // ... a compression the stage cannot decode: its decode job fails

#define FEAT_LZ4        (1ull << 17)
#define FEAT_COMPRESSED (1ull << 22)
#define FEAT_EMBED_DATA (1ull << 16)
// wire format "lz4-stage-v1": a 32-byte preamble in front of every DRR_BEGIN of a COMPRESS output
// (u64 magic "MTZLZ4W1", u32 version, u32 flags, 16 zero bytes), outside the stream checksum.  The
// host paths write and strip it; the kernels only see its one flag, carried in mtz_rec.resv of
// the BEGIN record: the original stream had the LZ4 feature flag.
#define WIRE_MAGIC      0x3157345A4C5A544DULL
#define WIRE_VERSION    1u
#define WIRE_PRE_BYTES  32u
#define WIRE_F_ORIG_LZ4 1u
#define WIRE_F_GZIP     2u      // COMPRESS with MTZ_FLAG_GZIP_WIRE or MTZ_FLAG_GZIP_ENCODE: gzip frames may
                                // follow.  Only a DECOMPRESS opened with MTZ_FLAG_GZIP_WIRE accepts the bit;
                                // any other refuses the preamble
#define ZIO_LZ4         15u

struct CodecRec {          // 32 B per record, device only
	uint64_t scratch;      // offset of this record's logical/encode scratch slot
	uint64_t out_off;      // offset of the output record
	uint32_t out_len;      // output payload bytes
	uint32_t flags;        // CF_*
	uint32_t need;         // scratch bytes reserved
	uint32_t pad;
};

struct CodecResult {       // device, mirrored to pinned host
	uint64_t out_bytes;    // running output offset after this batch
	uint32_t bad;          // first record whose frame failed to decode (0xffffffff none)
	uint32_t n_dec;        // records decoded
	uint32_t n_enc;        // records stored compressed on output
	uint32_t n_cert;       // ... of which certified (input frame == encoder output), not re-encoded
	uint32_t n_pass;       // COMPRESS with MTZ_FLAG_COMPRESSED_IN: LZ4 records forwarded as they are
	uint32_t n_lzjb;       // ... lzjb records decoded (not counted in n_dec)
	uint32_t n_zle;        // ... zle records decoded (likewise)
	uint32_t n_gzip;       // ... with MTZ_FLAG_GZIP_IN gzip records inflated (likewise); also DECOMPRESS
	                       // with MTZ_FLAG_GZIP_WIRE
	uint32_t n_gzpass;     // COMPRESS with MTZ_FLAG_GZIP_WIRE: gzip records forwarded (not in n_pass)
	uint32_t n_gz_enc;     // COMPRESS with MTZ_FLAG_GZIP_ENCODE: records stored as the stage's zlib frame
	                       // (not in n_enc)
};

// ---- plan, step 1: flags + scratch need -----------------------------------
// `cin`: COMPRESS with MTZ_FLAG_COMPRESSED_IN, `gzip`: ... and MTZ_FLAG_GZIP_IN, `gzwire`: the handle has
// MTZ_FLAG_GZIP_WIRE.  The one place that decides what becomes of a compressed DRR_WRITE: in COMPRESS
// with `cin` lzjb / zle, and gzip-1 .. gzip-9 with `gzip`, are decoded and offered to the encoder like
// a raw record, LZ4, and gzip-1 .. gzip-9 with `gzwire`, are forwarded as they are, any other
// compression fails the record (MTZ_ECODEC); in DECOMPRESS with `gzwire` gzip-1 .. gzip-9 are decoded
// (k_inflate) and leave raw.
#define ZIO_LZJB 3u
#define ZIO_ZLE  14u
#define ZIO_GZIP1 5u
#define ZIO_GZIP9 13u
__device__ __forceinline__ bool is_gzip(uint32_t comp) { return comp >= ZIO_GZIP1 && comp <= ZIO_GZIP9; }
__global__ void k_plan_need(const mtz_rec *__restrict__ recs, uint32_t n, uint32_t mode,
    CodecRec *__restrict__ cr, uint64_t *__restrict__ vals, bool cin = false, bool gzip = false,
    bool gzwire = false)
{
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n) return;
	const mtz_rec rec = recs[r];
	uint32_t f = 0;
	if (rec.type == DRR_WRITE_T) {
		f |= CF_WRITE;
		const bool gz = is_gzip(rec.comp);
		if ((rec.comp == ZIO_LZ4 && (mode == MTZ_MODE_DECOMPRESS || mode == MTZ_MODE_RECOMPRESS)) ||
		    (gzwire && gz && mode == MTZ_MODE_DECOMPRESS))
			f |= CF_DEC;
		if (cin && mode == MTZ_MODE_COMPRESS && rec.comp != 0u)
			f |= rec.comp == ZIO_LZJB || rec.comp == ZIO_ZLE || (gzip && gz) ? CF_DEC :
			     rec.comp == ZIO_LZ4 || (gzwire && gz) ? CF_PASS : CF_BAD;
		if ((mode == MTZ_MODE_COMPRESS || mode == MTZ_MODE_RECOMPRESS) &&
		    (rec.comp == 0u || (f & CF_DEC)))
			f |= CF_ENC;
	}
	const uint32_t need = (f & (CF_DEC | CF_ENC)) ? ((rec.lsize + 15u) & ~15u) + 16u : 0u;
	CodecRec c;
	c.scratch = 0; c.out_off = 0; c.out_len = 0; c.flags = f; c.need = need; c.pad = 0;
	cr[r] = c;
	vals[r] = need;
}

// ---- generic exclusive scan of u64 (single CTA, any n) --------------------
#define XSCAN_THREADS 1024
__global__ void __launch_bounds__(XSCAN_THREADS)
k_xscan_u64(const uint64_t *__restrict__ in, uint64_t *__restrict__ out, uint32_t n,
    uint64_t *total, const uint64_t *init)
{
	__shared__ uint64_t s_warp[XSCAN_THREADS / 32];
	__shared__ uint64_t s_run;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	if (threadIdx.x == 0) s_run = init ? *init : 0ull;
	__syncthreads();
	for (uint32_t base = 0; base < n; base += XSCAN_THREADS) {
		const uint32_t i = base + threadIdx.x;
		const uint64_t v = (i < n) ? in[i] : 0ull;
		uint64_t inc = v;
#pragma unroll
		for (int d = 1; d < 32; d <<= 1) {
			const uint64_t up = __shfl_up_sync(0xffffffffu, (unsigned long long)inc, d);
			if (lane >= d) inc += up;
		}
		if (lane == 31) s_warp[warp] = inc;
		__syncthreads();
		if (warp == 0) {
			uint64_t w = s_warp[lane];
#pragma unroll
			for (int d = 1; d < 32; d <<= 1) {
				const uint64_t up = __shfl_up_sync(0xffffffffu, (unsigned long long)w, d);
				if (lane >= d) w += up;
			}
			s_warp[lane] = w;
		}
		__syncthreads();
		const uint64_t run = s_run;
		const uint64_t wpre = warp ? s_warp[warp - 1] : 0ull;
		if (i < n) out[i] = run + wpre + inc - v;
		__syncthreads();
		if (threadIdx.x == 0) s_run = run + s_warp[XSCAN_THREADS / 32 - 1];
		__syncthreads();
	}
	if (threadIdx.x == 0 && total != nullptr) *total = s_run;
}

// ---- plan, step 2: jobs with absolute device addresses --------------------
// With `dec_gz` (DECOMPRESS with MTZ_FLAG_GZIP_WIRE) the decode job of a gzip record goes there and its
// slot of `dec` stays empty, so that K2, which decodes every job of `dec` with lsize != 0, never sees
// it; k_inflate runs over `dec_gz`, whose other slots are empty.
__global__ void k_plan_jobs(const uint8_t *__restrict__ d_in, const mtz_rec *__restrict__ recs,
    uint32_t n, CodecRec *__restrict__ cr, const uint64_t *__restrict__ offs,
    uint8_t *d_logical, uint8_t *d_enc, mtz_job *__restrict__ dec, mtz_job *__restrict__ enc,
    mtz_job *__restrict__ dec_gz = nullptr)
{
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n) return;
	const mtz_rec rec = recs[r];
	CodecRec c = cr[r];
	c.scratch = offs[r];
	cr[r] = c;
	const uint8_t *pay = d_in + rec.off + DRR_HDR;
	mtz_job jd, je;
	jd.src_off = jd.dst_off = 0; jd.src_len = 0; jd.lsize = 0; jd.out_len = 0; jd.status = 0;
	je = jd;
	if (c.flags & CF_BAD) {
		jd.status = MTZ_ECODEC;                 // no decoder for it
	} else if (c.flags & CF_DEC) {
		jd.src_off = (uint64_t)(uintptr_t)pay;
		jd.dst_off = (uint64_t)(uintptr_t)(d_logical + c.scratch);
		jd.src_len = rec.payload; jd.lsize = rec.lsize;
	}
	if (c.flags & CF_ENC) {
		je.src_off = (c.flags & CF_DEC) ? (uint64_t)(uintptr_t)(d_logical + c.scratch)
		                               : (uint64_t)(uintptr_t)pay;
		je.dst_off = (uint64_t)(uintptr_t)(d_enc + c.scratch);
		je.lsize = rec.lsize;
	}
	if (dec_gz != nullptr) {
		mtz_job none;
		none.src_off = none.dst_off = 0; none.src_len = 0; none.lsize = 0; none.out_len = 0; none.status = 0;
		const bool gz = is_gzip(rec.comp);
		dec_gz[r] = gz ? jd : none;
		if (gz) jd = none;
	}
	dec[r] = jd; enc[r] = je;
}

// ---- layout: output payload length per record -----------------------------
// `gz_enc` (COMPRESS with MTZ_FLAG_GZIP_ENCODE): k_deflate_from_lz4's jobs; a record leaves as its zlib
// frame (gzip-1, at gz_enc[r].dst_off) when gz_enc[r].out_len < enc[r].out_len, i.e. when that frame was
// written.
__device__ __forceinline__ bool gz_wins(const mtz_job *gz, const mtz_job *enc, uint32_t r)
{
	return gz != nullptr && gz[r].out_len < enc[r].out_len;
}

__global__ void k_layout(const mtz_rec *__restrict__ recs, uint32_t n, CodecRec *__restrict__ cr,
    const mtz_job *__restrict__ dec, const mtz_job *__restrict__ enc,
    uint64_t *__restrict__ vals, CodecResult *__restrict__ res, uint32_t rec_base,
    const uint32_t *__restrict__ cert = nullptr, const mtz_job *__restrict__ dec_gz = nullptr,
    const mtz_job *__restrict__ gz_enc = nullptr)
{
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n) return;
	const mtz_rec rec = recs[r];
	CodecRec c = cr[r];
	uint32_t len = rec.payload;
	if (c.flags & CF_BAD) atomicMin(&res->bad, r + rec_base);      // stays as it is: the batch fails
	const bool gz = is_gzip(rec.comp);
	if (c.flags & CF_DEC) {
		if ((dec_gz != nullptr && gz ? dec_gz[r] : dec[r]).status != MTZ_OK) atomicMin(&res->bad, r + rec_base);
		else atomicAdd(rec.comp == ZIO_LZJB ? &res->n_lzjb : rec.comp == ZIO_ZLE ? &res->n_zle :
		    gz ? &res->n_gzip : &res->n_dec, 1u);
		len = rec.lsize;
	}
	if (c.flags & CF_PASS) atomicAdd(gz ? &res->n_gzpass : &res->n_pass, 1u);
	if ((c.flags & CF_ENC) && enc[r].out_len < rec.lsize) {
		const bool g = gz_wins(gz_enc, enc, r);
		len = g ? gz_enc[r].out_len : enc[r].out_len;
		atomicAdd(g ? &res->n_gz_enc : &res->n_enc, 1u);
		if (cert != nullptr && cert[r] != 0u) atomicAdd(&res->n_cert, 1u);
	}
	c.out_len = len;
	cr[r] = c;
	vals[r] = (uint64_t)DRR_HDR + len;
}

// ---- assemble ---------------------------------------------------------------
template <typename V>
__device__ __forceinline__ void warp_copy_vec(uint8_t *dst, const uint8_t *src, uint32_t n, int lane)
{
	const uint32_t nv = n / (uint32_t)sizeof(V);
	const V *s = reinterpret_cast<const V *>(src);
	V *d = reinterpret_cast<V *>(dst);
	uint32_t i = (uint32_t)lane;
	for (; i + 96u < nv; i += 128u) {                   // 4 vectors in flight per lane
		const V a = s[i], b = s[i + 32u], c = s[i + 64u], e = s[i + 96u];
		d[i] = a; d[i + 32u] = b; d[i + 64u] = c; d[i + 96u] = e;
	}
	for (; i < nv; i += 32u) d[i] = s[i];
	for (uint32_t k = nv * (uint32_t)sizeof(V) + (uint32_t)lane; k < n; k += 32u) dst[k] = src[k];
}

__device__ __forceinline__ void warp_copy(uint8_t *dst, const uint8_t *src, uint32_t n, int lane)
{
	const uintptr_t a = (uintptr_t)dst | (uintptr_t)src;
	if ((a & 15u) == 0) warp_copy_vec<uint4>(dst, src, n, lane);
	else if ((a & 7u) == 0) warp_copy_vec<uint2>(dst, src, n, lane);
	else if ((a & 3u) == 0) warp_copy_vec<uint32_t>(dst, src, n, lane);
	else warp_copy_vec<uint8_t>(dst, src, n, lane);
}

#define ASM_THREADS 256
__global__ void __launch_bounds__(ASM_THREADS)
k_assemble(const uint8_t *__restrict__ d_in, const mtz_rec *__restrict__ recs, uint32_t n,
    uint32_t mode, CodecRec *__restrict__ cr, const uint64_t *__restrict__ out_offs,
    const mtz_job *__restrict__ enc, const uint8_t *d_logical, const uint8_t *d_enc,
    uint8_t *__restrict__ d_out, mtz_rec *__restrict__ out_recs,
    const uint32_t *__restrict__ cert = nullptr, const mtz_job *__restrict__ gz_enc = nullptr)
{
	const int lane = threadIdx.x & 31;
	const uint32_t gw = blockIdx.x * (ASM_THREADS / 32) + (threadIdx.x >> 5);
	const uint32_t nw = gridDim.x * (ASM_THREADS / 32);
	for (uint32_t r = gw; r < n; r += nw) {
		const mtz_rec rec = recs[r];
		const CodecRec c = cr[r];
		const uint64_t oo = out_offs[r];
		const uint8_t *hin = d_in + rec.off;
		uint8_t *hout = d_out + oo;
		// header: 78 words, both sides 4-byte aligned
		for (uint32_t i = (uint32_t)lane; i < DRR_HDR / 4u; i += 32u)
			reinterpret_cast<uint32_t *>(hout)[i] = reinterpret_cast<const uint32_t *>(hin)[i];
		__syncwarp();
		uint32_t ocomp = rec.comp;
		const uint8_t *psrc = hin + DRR_HDR;
		uint32_t ncopy = c.out_len;
		if (c.flags & CF_WRITE) {
			const bool enc_ok = (c.flags & CF_ENC) && enc[r].out_len < rec.lsize;
			if (enc_ok && gz_wins(gz_enc, enc, r)) {
				// the stage's zlib frame, zero-padded by k_deflate_from_lz4 itself
				psrc = reinterpret_cast<const uint8_t *>((uintptr_t)gz_enc[r].dst_off);
				ocomp = ZIO_GZIP1;
				if (lane == 0) {
					hout[50] = (uint8_t)ZIO_GZIP1;
					*reinterpret_cast<uint64_t *>(hout + 96) = (uint64_t)c.out_len;
				}
			} else if (enc_ok) {
				// certified (K3c): the frame is the input's own BE32(clen) + block, zero-padded
				const uint32_t cl = cert ? cert[r] : 0u;
				if (cl != 0u) ncopy = cl; else psrc = d_enc + c.scratch;
				ocomp = ZIO_LZ4;
				if (lane == 0) {
					hout[50] = (uint8_t)ZIO_LZ4;
					*reinterpret_cast<uint64_t *>(hout + 96) = (uint64_t)c.out_len;
				}
			} else if (c.flags & CF_DEC) {
				psrc = d_logical + c.scratch; ocomp = 0;
				if (lane == 0) {
					hout[50] = 0;
					*reinterpret_cast<uint64_t *>(hout + 96) = 0ull;
				}
			}
		} else if (rec.type == DRR_BEGIN_T && lane == 0) {
			uint64_t vi = *reinterpret_cast<const uint64_t *>(hin + 16);
			const uint64_t feat = (vi >> 2) & ((1ull << 30) - 1ull);
			(void)feat;
			if (mode == MTZ_MODE_COMPRESS) {
				vi |= (FEAT_COMPRESSED | FEAT_LZ4) << 2;
			} else if (mode == MTZ_MODE_DECOMPRESS) {
				vi &= ~((FEAT_COMPRESSED | FEAT_LZ4) << 2);
				if (rec.resv & WIRE_F_ORIG_LZ4) vi |= FEAT_LZ4 << 2;    // from the wire preamble
			} else if (mode == MTZ_MODE_RECOMPRESS) {
				vi |= (FEAT_COMPRESSED | FEAT_LZ4) << 2;
			}
			*reinterpret_cast<uint64_t *>(hout + 16) = vi;
		}
		warp_copy(hout + DRR_HDR, psrc, ncopy, lane);
		for (uint32_t i = ncopy + (uint32_t)lane; i < c.out_len; i += 32u) hout[DRR_HDR + i] = 0;
		if (lane == 0) {
			mtz_rec o;
			o.off = oo; o.payload = c.out_len; o.type = rec.type;
			o.lsize = rec.lsize; o.comp = ocomp; o.resv = 0;
			out_recs[r] = o;
		}
	}
}

// ---- stamp: dump_record() chain over the output ---------------------------
// The transform of the running checksum by a stamped record is NOT affine: the 8
// words folded in after the header are the 32-bit halves of the running value
// itself.  It is still "affine plus a linear form of the halves".  With
//   x_r   = value stamped into record r (running checksum after its 280 header bytes)
//   w_0..7 = the 32-bit halves of x_r
//   Q_r   = zero-state sums of [payload of r | header words of r+1], n2 words
// the next stamp is (word w_k sits n2 + 8 - k words from the end of the segment)
//   x_{r+1} = apply(x_r, N = n2 + 8) + sum_k T_j(n2 + 8 - k) w_k + Q_r
// so everything except 3 + 8 multiply-adds per component is computed for all records
// in parallel (k_stamp_prep) and the serial walk is one step of independent
// multiply-adds per record, split over four lanes (one per component a, b, c, d) that
// exchange the new value by shuffle.  BEGIN records (checksum field is data, running
// value restarts), END records (the running value is also written into the payload-less
// END header, which changes that header's sums) and the batch edges take the generic
// path.  This replaced a one-lane recurrence that walked every record through the full
// Fletcher update.
// Folded once more: x.a .. x.d ARE the halves (x_i = w_2i + 2^32 w_2i+1), so the apply() part
// multiplies the same eight words -- component j of x_{r+1} is ONE linear form of w_0..w_7 plus a
// constant, with 64-bit weights  C_k = T_j(n2+8-k) + E_j,i  (k = 2i)  or  + (E_j,i << 32)  (k = 2i+1),
// E = [[1],[N,1],[T2N,N,1],[T3N,T2N,N,1]]: eight 64x32-bit multiply-adds per lane and step.
struct alignas(16) StampStep {          // transition x_r -> x_{r+1}; 304 B
	uint64_t c[4][9];         // lane j: weights of w_0..w_7 | constant
	uint64_t woff;            // byte offset in d_out of record r+1's checksum field
	uint32_t fast, pad;
};

__global__ void k_stamp_prep(const mtz_rec *__restrict__ out_recs, const RecSums *__restrict__ osums,
    uint32_t n, StampStep *__restrict__ steps)
{
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n) return;
	bool fast = false;
	if (r + 1u < n) {
		const uint32_t t1 = osums[r + 1u].type;
		fast = (t1 != DRR_BEGIN_T && t1 != DRR_END_T);
	}
	StampStep *o = &steps[r];
	if (!fast) { o->fast = 0; o->pad = 0; o->woff = 0; return; }
	const RecSums rs = osums[r];
	const Ck4 nh = osums[r + 1u].head;
	const uint64_t n2 = rs.nbody + DRR_CKOFF / 4u, N = n2 + 8u;
	const Part b = { rs.nbody, rs.body.a, rs.body.b, rs.body.c, rs.body.d };
	const Part hd = { DRR_CKOFF / 4u, nh.a, nh.b, nh.c, nh.d };
	const Part q = concat(b, hd);
	uint64_t g[4] = { q.a, q.b, q.c, q.d };
	uint64_t W[4][8];
#pragma unroll
	for (int k = 0; k < 8; k++) {
		const uint64_t x = n2 + 8u - (uint64_t)k;
		W[0][k] = 1; W[1][k] = x; W[2][k] = tri2(x); W[3][k] = tri3(x);
	}
	if (rs.type == DRR_BEGIN_T) {
		// bytes 280..311 of a BEGIN header are data: their contribution is a constant
		const uint64_t e[4] = { rs.emb.a, rs.emb.b, rs.emb.c, rs.emb.d };
#pragma unroll
		for (int j = 0; j < 4; j++) {
#pragma unroll
			for (int k = 0; k < 8; k++) {
				const uint64_t w = (k & 1) ? (e[k >> 1] >> 32) : (uint64_t)(uint32_t)e[k >> 1];
				g[j] += W[j][k] * w;
				W[j][k] = 0;
			}
		}
	}
	const uint64_t t2 = tri2(N), t3 = tri3(N);
	const uint64_t E[4][4] = { { 1, 0, 0, 0 }, { N, 1, 0, 0 }, { t2, N, 1, 0 }, { t3, t2, N, 1 } };
#pragma unroll
	for (int j = 0; j < 4; j++) {
#pragma unroll
		for (int k = 0; k < 8; k++)
			o->c[j][k] = W[j][k] + ((k & 1) ? (E[j][k >> 1] << 32) : E[j][k >> 1]);
		o->c[j][8] = g[j];
	}
	o->woff = out_recs[r + 1u].off + DRR_CKOFF;
	o->fast = 1; o->pad = 0;
}

// value stamped into record r given the running checksum s that precedes it (generic path)
__device__ __forceinline__ Ck4 stamp_enter(Ck4 s, uint8_t *__restrict__ d_out,
    const mtz_rec *__restrict__ out_recs, const RecSums *__restrict__ osums, uint32_t r,
    ScanResult *__restrict__ res, int lane)
{
	const RecSums rs = osums[r];
	uint8_t *hdr = d_out + out_recs[r].off;
	Ck4 head = rs.head;
	if (rs.type == DRR_BEGIN_T) s.a = s.b = s.c = s.d = 0;
	if (rs.type == DRR_END_T) {
		if (lane == 0) {
			uint64_t *e = reinterpret_cast<uint64_t *>(hdr + 8);
			e[0] = s.a; e[1] = s.b; e[2] = s.c; e[3] = s.d;
			res->end_ck = s; res->end_seen = 1;
		}
		// the END header changed under the sums K1 took: redo its 70 words
		Ck4 t = { 0, 0, 0, 0 };
		const uint32_t *w = reinterpret_cast<const uint32_t *>(hdr);
		for (uint32_t i = 0; i < DRR_CKOFF / 4u; i++) {
			uint32_t v;
			if (i >= 2u && i < 10u) {            // bytes 8..39 just written
				const uint64_t q = (i < 4u) ? s.a : (i < 6u) ? s.b : (i < 8u) ? s.c : s.d;
				v = (i & 1u) ? (uint32_t)(q >> 32) : (uint32_t)q;
			} else {
				v = w[i];
			}
			t.a += v; t.b += t.a; t.c += t.b; t.d += t.c;
		}
		head = t;
	}
	const Part h = { DRR_CKOFF / 4u, head.a, head.b, head.c, head.d };
	const Ck4 x = apply(s, h);
	if (rs.type != DRR_BEGIN_T && lane == 0) {
		uint64_t *ck = reinterpret_cast<uint64_t *>(hdr + DRR_CKOFF);
		ck[0] = x.a; ck[1] = x.b; ck[2] = x.c; ck[3] = x.d;
	}
	return x;
}

// running checksum after record r given the value x stamped into it (generic path)
__device__ __forceinline__ Ck4 stamp_leave(const Ck4 &x, const RecSums *__restrict__ osums, uint32_t r)
{
	const RecSums rs = osums[r];
	Ck4 s = fold_cksum_words(x, rs.type == DRR_BEGIN_T ? rs.emb : x);
	const Part b = { rs.nbody, rs.body.a, rs.body.b, rs.body.c, rs.body.d };
	return apply(s, b);
}

// keep a 64-bit value in its register at this point (defeats re-association across it)
#ifdef MTZ_HOST_EMUL
#define MTZ_PIN64(x) do { } while (0)
#else
#define MTZ_PIN64(x) asm volatile("" : "+l"(x))
#endif
#define STAMP_GROUP   32
#define STAMP_THREADS 128
#define STAMP_LOADERS (STAMP_THREADS / 32 - 1)
// warp 0 walks the chain; warps 1..3 stage the next STAMP_GROUP transitions (12.8 KB) into shared
// memory.  One loader warp with one load in flight per lane could not keep up with the chain:
// three warps, four loads in flight per lane
__global__ void __launch_bounds__(STAMP_THREADS)
k_stamp_chain(uint8_t *__restrict__ d_out, const mtz_rec *__restrict__ out_recs,
    const RecSums *__restrict__ osums, const StampStep *__restrict__ steps, uint32_t n,
    Ck4 *__restrict__ carry_out, ScanResult *__restrict__ res)
{
	__shared__ StampStep s_steps[2][STAMP_GROUP + 1];     // +1: the weight prefetch of step i+1 needs no bounds check
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int j = lane & 3;
	if (n == 0u) return;
	const uint32_t T = n - 1u;                                    // transitions
	const uint32_t ngroups = (T + STAMP_GROUP - 1u) / STAMP_GROUP;
	constexpr uint32_t V4 = (uint32_t)(sizeof(StampStep) / sizeof(uint4));
	auto stage = [&](uint32_t g) {
		const uint32_t r0 = g * STAMP_GROUP, cnt = min((uint32_t)STAMP_GROUP, T - r0);
		const uint4 *src = reinterpret_cast<const uint4 *>(steps + r0);
		uint4 *dst = reinterpret_cast<uint4 *>(&s_steps[g & 1u][0]);
		const uint32_t nv = cnt * V4, stride = 32u * STAMP_LOADERS;
		for (uint32_t i = (uint32_t)(warp - 1) * 32u + (uint32_t)lane; i < nv; i += 4u * stride) {
			uint4 t0, t1, t2, t3;                      // four independent loads in flight
			const uint32_t i1 = i + stride, i2 = i + 2u * stride, i3 = i + 3u * stride;
			t0 = src[i];
			if (i1 < nv) t1 = src[i1];
			if (i2 < nv) t2 = src[i2];
			if (i3 < nv) t3 = src[i3];
			dst[i] = t0;
			if (i1 < nv) dst[i1] = t1;
			if (i2 < nv) dst[i2] = t2;
			if (i3 < nv) dst[i3] = t3;
		}
	};
	if (warp >= 1 && ngroups > 0u) stage(0);
	__syncthreads();

	Ck4 x = { 0, 0, 0, 0 };
	uint64_t own = 0;
	if (warp == 0) {
		x = stamp_enter(*carry_out, d_out, out_recs, osums, 0u, res, lane);
		own = (j == 0) ? x.a : (j == 1) ? x.b : (j == 2) ? x.c : x.d;
	}
	for (uint32_t g = 0; g < ngroups; g++) {
		if (warp >= 1) {
			if (g + 1u < ngroups) stage(g + 1u);
		} else {
			const uint32_t r0 = g * STAMP_GROUP, cnt = min((uint32_t)STAMP_GROUP, T - r0);
			// The weights of transition i+1 are loaded from shared memory (29 cycles) while transition
			// i is computed; two register sets alternate so that no value is ever copied.
			const StampStep *sg = &s_steps[g & 1u][0];
			uint64_t ca[9], cb[9];
			uint64_t woa = sg[0].woff, wob = 0;
			uint32_t fa = sg[0].fast, fb = 0;
#pragma unroll
			for (int q = 0; q < 9; q++) { ca[q] = sg[0].c[j][q]; cb[q] = 0; }
#define STAMP_STEP(C, WOFF, FAST, NC, NWOFF, NFAST, IDX)                                         \
			{                                                                                    \
				const uint32_t i_ = (IDX);                                                       \
				{                                                                                \
					const StampStep &nx = sg[i_ + 1u];       /* (slot 32 is padding) */          \
					_Pragma("unroll") for (int q = 0; q < 9; q++) NC[q] = nx.c[j][q];            \
					NWOFF = nx.woff; NFAST = nx.fast;                                            \
				}                                                                                \
				const uint32_t lo = (uint32_t)own, hi = (uint32_t)(own >> 32);                   \
				const uint32_t w0 = __shfl_sync(0xffffffffu, lo, 0), w1 = __shfl_sync(0xffffffffu, hi, 0); \
				const uint32_t w2 = __shfl_sync(0xffffffffu, lo, 1), w3 = __shfl_sync(0xffffffffu, hi, 1); \
				const uint32_t w4 = __shfl_sync(0xffffffffu, lo, 2), w5 = __shfl_sync(0xffffffffu, hi, 2); \
				const uint32_t w6 = __shfl_sync(0xffffffffu, lo, 3), w7 = __shfl_sync(0xffffffffu, hi, 3); \
				if (FAST != 0u) {                                                                \
					/* four independent multiply-add chains (pinned: left alone the compiler     \
					 * folds them into ONE dependent chain of ~10 cycles per term) */            \
					uint64_t p0 = C[8] + C[0] * (uint64_t)w0 + C[1] * (uint64_t)w1;              \
					uint64_t p1 = C[2] * (uint64_t)w2 + C[3] * (uint64_t)w3;                     \
					uint64_t p2 = C[4] * (uint64_t)w4 + C[5] * (uint64_t)w5;                     \
					uint64_t p3 = C[6] * (uint64_t)w6 + C[7] * (uint64_t)w7;                     \
					MTZ_PIN64(p0); MTZ_PIN64(p1); MTZ_PIN64(p2); MTZ_PIN64(p3);                  \
					own = (p0 + p1) + (p2 + p3);                                                 \
					/* every lane stores (lanes 4..31 repeat lanes 0..3): no divergent branch */   \
					*reinterpret_cast<uint64_t *>(d_out + WOFF + 8u * (uint32_t)j) = own;        \
				} else {                                                                         \
					x.a = ((uint64_t)w1 << 32) | w0; x.b = ((uint64_t)w3 << 32) | w2;            \
					x.c = ((uint64_t)w5 << 32) | w4; x.d = ((uint64_t)w7 << 32) | w6;            \
					const Ck4 s_ = stamp_leave(x, osums, r0 + i_);                               \
					x = stamp_enter(s_, d_out, out_recs, osums, r0 + i_ + 1u, res, lane);        \
					own = (j == 0) ? x.a : (j == 1) ? x.b : (j == 2) ? x.c : x.d;                \
				}                                                                                \
			}
			uint32_t i = 0;
			for (; i + 1u < cnt; i += 2u) {
				STAMP_STEP(ca, woa, fa, cb, wob, fb, i)
				STAMP_STEP(cb, wob, fb, ca, woa, fa, i + 1u)
			}
			if (i < cnt) STAMP_STEP(ca, woa, fa, cb, wob, fb, i)
#undef STAMP_STEP
		}
		__syncthreads();
	}
	if (warp == 0) {
		const uint32_t lo = (uint32_t)own, hi = (uint32_t)(own >> 32);
		x.a = ((uint64_t)__shfl_sync(0xffffffffu, hi, 0) << 32) | __shfl_sync(0xffffffffu, lo, 0);
		x.b = ((uint64_t)__shfl_sync(0xffffffffu, hi, 1) << 32) | __shfl_sync(0xffffffffu, lo, 1);
		x.c = ((uint64_t)__shfl_sync(0xffffffffu, hi, 2) << 32) | __shfl_sync(0xffffffffu, lo, 2);
		x.d = ((uint64_t)__shfl_sync(0xffffffffu, hi, 3) << 32) | __shfl_sync(0xffffffffu, lo, 3);
		const Ck4 s = stamp_leave(x, osums, n - 1u);
		if (lane == 0) { *carry_out = s; res->carry = s; }
	}
}

} // namespace mtz
