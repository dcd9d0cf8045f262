/*
 * manatee_gpu.h -- C ABI of libmanatee_gpu.so, the H100 snapshot-stream stage.
 *
 * This is the drop-in boundary for the one bulk-data path of
 * TritonDataCenter/manatee: the ZFS-send byte stream that the sender pumps
 * with   zfsSend.stdout.pipe(socket)        (lib/backupSender.js:179)
 * and the receiver with   socket.pipe(zfsRecv.stdin)   (lib/zfsClient.js:826).
 * The reference has no FFI for this path (it is two Node .pipe() calls); the
 * entry points below are what an N-API addon for a `stream.Transform` spliced
 * into those two pipes binds (INTEGRATION.md shows the binding and the two
 * one-line patches).  Plain pointers and sizes only, no torch/CUDA types.
 *
 * Threading: one producer thread (ring_acquire/commit/write/flush) and one
 * consumer thread (out_peek/out_consume/read) per handle; handles are
 * independent.  Every call returns 0 (MTZ_OK) or a negative MTZ_E* code; the
 * message for the last failure on a handle is mtz_last_error(h).  A failure
 * is sticky: once a handle has failed every later call returns the same code,
 * which the JS stage turns into destroy(err) => job.done='failed' exactly like
 * a non-zero `zfs send` exit (lib/backupSender.js:214-221) or a `zfs recv`
 * failure (lib/zfsClient.js:808-815, 867-876).
 */
#ifndef MANATEE_GPU_H
#define MANATEE_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MTZ_ABI_VERSION 2

/* ---- return codes ---- */
#define MTZ_OK        0
#define MTZ_EINVAL   -1   /* bad argument / bad state */
#define MTZ_EAGAIN   -2   /* would block: ring full (producer) or empty (consumer) */
#define MTZ_ECUDA    -3   /* CUDA runtime failure, see mtz_last_error */
#define MTZ_EFORMAT  -4   /* malformed send stream (bad magic / type / length) */
#define MTZ_ECKSUM   -5   /* embedded or END Fletcher-4 mismatch (like zfs recv ECKSUM) */
#define MTZ_ECODEC   -6   /* LZ4 frame does not decode to drr_logical_size */
#define MTZ_ENOSPC   -7   /* output capacity exceeded */
#define MTZ_ENOMEM   -8
#define MTZ_EOF      -9   /* consumer: stream finished and fully drained */
#define MTZ_ENOGPU  -10   /* no usable sm_90 device: there is NO CPU fallback */
#define MTZ_ECANCELED -11 /* mtz_cancel(): the pipe was torn down from outside */

/* ---- stage modes ---- */
#define MTZ_MODE_VERIFY      0  /* identity bytes; every stream checksum verified */
#define MTZ_MODE_COMPRESS    1  /* sender: raw DRR_WRITE payload -> ZFS-LZ4, re-stamp */
#define MTZ_MODE_DECOMPRESS  2  /* receiver: exact inverse of COMPRESS */
#define MTZ_MODE_RECOMPRESS  3  /* decode LZ4 records, verify, re-encode, re-stamp */
#define MTZ_MODE_PASSTHROUGH 4  /* rings + H2D/D2H only, no parsing (plumbing tests) */

/* config flags */
#define MTZ_FLAG_DEFER_VERIFY 1u /* shard mode: mtz_process_host only accumulates per-record
                                  * sums; verdict comes from mtz_dev_aggregate/mtz_dev_finish
                                  * once the preceding shards' checksum is known */

#define MTZ_FLAG_REENCODE_ALL 2u /* RECOMPRESS: run the encoder on every record.  Default: a record whose
                                  * incoming LZ4 block is PROVEN to be the encoder's own output for the
                                  * decoded bytes is passed through (mtz_stats.lz4_certified counts them);
                                  * the output bytes are the same either way */

#define MTZ_FLAG_BLOCK_CKSUM 4u  /* VERIFY / COMPRESS / DECOMPRESS / RECOMPRESS (not PASSTHROUGH): check every
                                  * DRR_WRITE against the on-disk block checksum `zfs send` copies into it
                                  * (drr_key, fletcher4 keys only).  A block stored raw on disk must match
                                  * its logical bytes: a mismatch fails the handle with MTZ_ECKSUM like a
                                  * stream checksum.  A block stored LZ4 on disk is compared with the
                                  * frame at hand: a mismatch is only counted (mtz_block_stats.frame_miss).
                                  * Counters: mtz_get_block_stats */

#define MTZ_FLAG_BLOCK_SHA256 8u /* with MTZ_FLAG_BLOCK_CKSUM only (MTZ_EINVAL without it): also check the
                                  * records whose key is a SHA-256 (drr_checksumtype 8, checksum=sha256),
                                  * by the same rules and with the same consequences as fletcher4 keys;
                                  * mtz_block_stats.sha256 counts them.  Without this flag they are skipped */

#define MTZ_FLAG_BLOCK_SHA512 16u /* with MTZ_FLAG_BLOCK_CKSUM only (MTZ_EINVAL without it), independent of
                                  * MTZ_FLAG_BLOCK_SHA256: also check the records whose key is a SHA-512/256
                                  * (drr_checksumtype 11, checksum=sha512), by the same rules and with the
                                  * same consequences as fletcher4 keys; mtz_block_stats.sha512 counts them.
                                  * Without this flag they are skipped */

#define MTZ_FLAG_BLOCK_FRAMES 32u /* with MTZ_FLAG_BLOCK_CKSUM only (MTZ_EINVAL without it), with or without the
                                  * SHA flags.  VERIFY: a DRR_WRITE that arrives raw while its key covers an
                                  * LZ4 frame on disk (otherwise skipped) gets a frame from the stage's
                                  * encoder, compared with the key by the rules COMPRESS applies to its own
                                  * output: frame_ok, or frame_miss (counted, never an error).  The output
                                  * bytes do not change.  mtz_block_stats.frames_encoded counts these
                                  * frames; with this flag and batch_bytes 0 VERIFY batches are 256 MiB.
                                  * The other modes accept the flag and do not change */

#define MTZ_FLAG_BLOCK_LZJB 64u  /* with MTZ_FLAG_BLOCK_CKSUM only (MTZ_EINVAL without it), with or without
                                  * BLOCK_FRAMES and the SHA flags.  Keys over an lzjb (on-disk compression 3)
                                  * or zle (14) frame are checked, otherwise skipped.  VERIFY and RECOMPRESS:
                                  * a record that arrives as that frame (send -c) is compared as it is.
                                  * VERIFY: a record that arrives raw gets a frame from the stage's lzjb / zle
                                  * encoder (ZFS's, at buffer address phase 0).  Either way the verdict is
                                  * frame_ok or frame_miss (counted, never an error) and the output bytes do
                                  * not change.  mtz_block_stats.lzjb_encoded / zle_encoded count the frames
                                  * encoded; with this flag and batch_bytes 0 VERIFY batches are 256 MiB.
                                  * COMPRESS and DECOMPRESS accept the flag and do not change without
                                  * MTZ_FLAG_BLOCK_LOGICAL */

#define MTZ_FLAG_BLOCK_LOGICAL 128u /* with MTZ_FLAG_BLOCK_CKSUM only (MTZ_EINVAL without it), with or without the
                                  * other block flags.  COMPRESS / DECOMPRESS / RECOMPRESS also check keys from
                                  * the logical bytes they hold (the raw input payload, or the decoder's
                                  * output for a record that arrives LZ4), so that a transfer over the
                                  * compressed wire counts what VERIFY counts on the raw stream.
                                  * RECOMPRESS: a block stored raw on disk that arrives LZ4 must match its
                                  * decoded bytes (MTZ_ECKSUM otherwise, as in DECOMPRESS).  With
                                  * MTZ_FLAG_BLOCK_LZJB: a record with an lzjb / zle key that arrives raw, or
                                  * LZ4 in DECOMPRESS / RECOMPRESS (COMPRESS decodes nothing), gets a frame from the stage's lzjb / zle encoder as in VERIFY
                                  * (frame_ok or frame_miss; lzjb_encoded / zle_encoded).  DECOMPRESS: a
                                  * record with an LZ4 key that arrives raw is the frame_miss COMPRESS
                                  * counted for it at the sender.  The output bytes and mtz_stats do not
                                  * change; mtz_block_stats.logical_checked counts these records.  VERIFY
                                  * accepts the flag and does not change */

typedef struct mtz_handle mtz_handle;

#define MTZ_MAX_DEVICES 16
#define MTZ_MAX_PEERS   16

typedef struct mtz_config {
	uint32_t struct_size;   /* sizeof(mtz_config), for ABI growth (v1 callers stop after n_slots) */
	int32_t  device;        /* CUDA ordinal (ignored when n_devices > 0) */
	uint32_t mode;          /* MTZ_MODE_* */
	uint32_t flags;         /* MTZ_FLAG_* */
	uint64_t ring_bytes;    /* pinned input ring (0 = max(256 MiB, 2 x batch_bytes)) */
	uint64_t out_ring_bytes;/* pinned output ring, codec modes (0 = ring_bytes) */
	uint64_t batch_bytes;   /* target bytes per GPU batch (0 = 32 MiB; 256 MiB in codec modes and
	                         * with MTZ_FLAG_BLOCK_FRAMES or MTZ_FLAG_BLOCK_LZJB) */
	uint32_t record_bytes;  /* expected recordsize hint (0 = 131072) */
	uint32_t n_slots;       /* batches in flight PER DEVICE (0 = 4) */
	/* ---- ABI v2: the GPUs of one box as ONE stage.  The stream is cut into whole-record
	 * batches and batch b runs on devices[b % n_devices] (record-index partition); the only
	 * thing that crosses between GPUs on the single-consumer path is the 64 bytes of running
	 * checksums that hop with the batches.  The reference serves N peers with N independent
	 * `zfs send`s (one _send per 'push', lib/backupSender.js:72-73); here one pass over the
	 * stream feeds every attached peer (mtz_fanout_attach). ---- */
	uint32_t n_devices;     /* 0 = just `device` */
	int32_t  devices[MTZ_MAX_DEVICES];
} mtz_config;

typedef struct mtz_stats {
	uint64_t bytes_in;      /* stream bytes accepted */
	uint64_t bytes_out;     /* stream bytes made available to the consumer */
	uint64_t records;       /* DRR records processed */
	uint64_t write_records; /* DRR_WRITE records */
	uint64_t lz4_decoded;   /* records LZ4-decoded */
	uint64_t lz4_encoded;   /* records stored LZ4-compressed on output */
	uint64_t batches;       /* GPU batches completed */
	uint64_t bad_record;    /* index of the first failing record, ~0 if none */
	uint64_t kernel_launches;
	double   gpu_ms;        /* sum of per-batch device time (CUDA events) */
	uint64_t end_seen;      /* DRR_END processed */
	double   k1_ms;         /* device time of the Fletcher-4 sums kernel (CUDA events) */
	double   codec_ms;      /* device time of the LZ4 kernels */
	uint64_t k1_launches;
	double   k3_ms;         /* device time of the LZ4 encode kernel alone (CUDA events) */
	uint64_t k3_launches;
	uint64_t lz4_certified; /* RECOMPRESS: records whose input frame was PROVEN to be the encoder's output
	                           (kernels_lz4.cuh warp_lz4_certify) and passed through; the rest were re-encoded */
} mtz_stats;

/* MTZ_FLAG_BLOCK_CKSUM counters (all zero with the flag off).  A DRR_WRITE whose key the stage
 * cannot check (not fletcher4 -- or sha256 with MTZ_FLAG_BLOCK_SHA256, sha512 with MTZ_FLAG_BLOCK_SHA512 --,
 * no key, encrypted, another on-disk compression, or no bytes at hand that the key covers) counts as
 * skipped. */
typedef struct mtz_block_stats {
	uint32_t struct_size;       /* sizeof(mtz_block_stats), set by the caller */
	uint32_t pad;
	uint64_t logical_ok;        /* stored raw on disk: logical bytes match the key */
	uint64_t frame_ok;          /* stored compressed on disk: the frame at hand matches the key */
	uint64_t frame_miss;        /* ... does not: another encoder wrote the disk block */
	uint64_t skipped;
	uint64_t first_frame_miss;  /* stream index of the first frame miss, ~0 if none */
	uint64_t sha256;            /* MTZ_FLAG_BLOCK_SHA256: records compared by SHA-256 (also counted above,
	                               or the cause of the failure) */
	uint64_t sha512;            /* MTZ_FLAG_BLOCK_SHA512: records compared by SHA-512/256 (likewise) */
	uint64_t frames_encoded;    /* MTZ_FLAG_BLOCK_FRAMES: frames encoded for the check (also counted in
	                               frame_ok / frame_miss, and in sha256 / sha512 where those hashed it) */
	uint64_t lzjb_encoded;      /* MTZ_FLAG_BLOCK_LZJB: lzjb frames encoded for the check (likewise) */
	uint64_t zle_encoded;       /* MTZ_FLAG_BLOCK_LZJB: zle frames encoded for the check (likewise) */
	uint64_t logical_checked;   /* MTZ_FLAG_BLOCK_LOGICAL: records compared thanks to that flag (also counted
	                               in logical_ok / frame_ok / frame_miss, or the cause of the failure) */
} mtz_block_stats;

/* One DRR record as seen by the kernels (32 B, little endian). */
typedef struct mtz_rec {
	uint64_t off;      /* byte offset of the 312-byte header in the batch */
	uint32_t payload;  /* payload bytes that follow the header */
	uint32_t type;     /* drr_type */
	uint32_t lsize;    /* DRR_WRITE: drr_logical_size, else 0 */
	uint32_t comp;     /* DRR_WRITE: drr_compressiontype, else 0 */
	uint64_t resv;
} mtz_rec;

/* One codec job (32 B): a frame to decode or a logical block to encode.
 * Offsets are relative to the src/dst base pointers of the call. */
typedef struct mtz_job {
	uint64_t src_off;  /* decode: BE32-framed LZ4 payload; encode: logical bytes */
	uint64_t dst_off;  /* decode: lsize bytes out; encode: frame slot of lsize bytes */
	uint32_t src_len;  /* decode: payload (psize) bytes; encode: unused */
	uint32_t lsize;    /* drr_logical_size */
	uint32_t out_len;  /* decode: lsize; encode: psize, or lsize = store raw */
	int32_t  status;   /* MTZ_OK or MTZ_ECODEC */
} mtz_job;

/* ---- lifecycle ----
 * One handle per spliced pipe, i.e. per `zfs send` child on the sender
 * (spawn at lib/backupSender.js:177) or per `zfs recv` child on the receiver
 * (spawn at lib/zfsClient.js:793); opened when the child is spawned, closed when
 * the pipe ends or fails. */
int32_t     mtz_abi_version(void);
int32_t     mtz_device_count(void);                 /* sm_90 devices visible, <0 on error */
int32_t     mtz_open(const mtz_config *cfg, mtz_handle **out);
int32_t     mtz_close(mtz_handle *h);
const char *mtz_last_error(mtz_handle *h);          /* h may be NULL: last open() error */
const char *mtz_strerror(int32_t code);

/* ---- streaming API over pinned rings (what the N-API Transform binds) ---- */
/* producer side == Transform._write(chunk): replaces the data path of
 * zfsSend.stdout.pipe(...) (lib/backupSender.js:179) / socket.pipe(...)
 * (lib/zfsClient.js:826).  acquire returns a slice of the PINNED input ring
 * (read(2)/memcpy straight into it), commit publishes n bytes of it. */
int32_t mtz_ring_acquire(mtz_handle *h, size_t want, void **ptr, size_t *got);
int32_t mtz_ring_commit(mtz_handle *h, size_t n);
int32_t mtz_write(mtz_handle *h, const void *buf, size_t n, int32_t block);
/* end of input == Transform._flush(): like stdout 'end' on the zfs send child.  A stream that
 * stops inside a record, or after whole records but before the DRR_END of an open sub-stream
 * (what a dying `zfs send` leaves), fails the handle with MTZ_EFORMAT. */
int32_t mtz_flush(mtz_handle *h);
/* consumer side == Transform.push(): processed stream bytes, in stream order */
int32_t mtz_out_peek(mtz_handle *h, const void **ptr, size_t *n);
int32_t mtz_out_consume(mtz_handle *h, size_t n);
int32_t mtz_read(mtz_handle *h, void *buf, size_t cap, size_t *got, int32_t block);
/* fd that becomes readable when output or an error is pending (eventfd): the
 * addon's uv_poll_t / napi_threadsafe_function wake-up source */
int32_t mtz_event_fd(mtz_handle *h);

/* ---- fan-out: several peers bootstrapping from the same snapshot share ONE pass.  Attach
 * every peer before the first input byte.  Each peer owns a pinned output ring fed from its
 * egress GPU devices[peer % n_devices] (one PCIe link / NIC queue per peer); in the re-encoding
 * modes the processed batch reaches the egress GPUs by an NCCL broadcast over NVLink from the
 * GPU that produced it (library-owned communicator), in VERIFY the verified input ring is shared
 * in place.  mtz_out_peek/consume are the peer-0 forms.  Replaces: one socket per _send,
 * lib/backupSender.js:166-179. ---- */
int32_t mtz_fanout_attach(mtz_handle *h, int32_t peer_id);
int32_t mtz_out_peek_peer(mtz_handle *h, int32_t peer_id, const void **ptr, size_t *n);
int32_t mtz_out_consume_peer(mtz_handle *h, int32_t peer_id, size_t n);
/* blocking read for one peer (mtz_read is the peer-0 form) */
int32_t mtz_read_peer(mtz_handle *h, int32_t peer_id, void *buf, size_t cap, size_t *got, int32_t block);
/* tear the pipe down from outside (socket error, stage.destroy()): fails the handle with
 * MTZ_ECANCELED and wakes every blocked mtz_write / mtz_read, like the reference's
 * zfsSend.kill() on a socket 'error' (lib/backupSender.js:230-233) */
int32_t mtz_cancel(mtz_handle *h);

/* counters for the job object the sender publishes through GET /backup/:uuid
 * (lib/backupServer.js:100-131 serialises the same object the sender mutates,
 * lib/backupSender.js:197-212): additive `job.gpu`, never read by the reference */
int32_t mtz_get_stats(mtz_handle *h, mtz_stats *st);
/* fills min(st->struct_size, sizeof(mtz_block_stats)) bytes */
int32_t mtz_get_block_stats(mtz_handle *h, mtz_block_stats *st);
/* running Fletcher-4 of the OUTPUT stream before DRR_END (== drr_end.drr_checksum) */
int32_t mtz_end_checksum(mtz_handle *h, uint64_t out[4]);

/* ---- bulk host API: a whole stream (or a whole-record slice of one) already in
 * host memory; internally pipelined H2D -> kernels -> D2H over n_slots streams.
 * in/out should come from mtz_host_alloc (pinned) for full PCIe rate.  Same
 * bytes-in / bytes-out contract as the two pipes above for a caller that holds the
 * stream in memory instead of a socket (bench.py's `e2e`, the shard drivers). ---- */
int32_t mtz_host_alloc(size_t bytes, void **ptr);
int32_t mtz_host_free(void *ptr);
int32_t mtz_process_host(mtz_handle *h, const void *in, size_t n, void *out,
    size_t out_cap, size_t *out_n);

/* ---- device-resident API (HBM in, HBM out): multi-GPU shards and kernel timing.
 * Pointers are CUDA device pointers passed as integers-in-void*.  The reference
 * serves N concurrent peers with N independent sends of the same snapshot
 * (one `_send` per 'push', lib/backupSender.js:72-73); here one stream is cut by
 * record index across GPUs and the only exchange is the 40-byte aggregate below
 * (SURVEY.md 8e).  The arithmetic itself replaces what the host OS's ZFS does
 * inside `zfs send` / `zfs recv` ([EXTERNAL] dmu_send.c dump_record(),
 * dmu_recv.c receive_read_record(), zfs_fletcher.c, lz4.c). ---- */
/* host-side DRR parse: fills recs[] for whole records in [buf, buf+n) */
int32_t mtz_index_host(const void *buf, size_t n, mtz_rec *recs, size_t cap,
    size_t *nrec, size_t *consumed);
/* GPU-side DRR parse of a resident stream (speculative strided header walk):
 * fills d_recs (device) for the whole records in [d_in, d_in+n); synchronises. */
int32_t mtz_dev_index(mtz_handle *h, const void *d_in, size_t n, mtz_rec *d_recs,
    size_t cap, size_t *nrec, size_t *consumed, void *cuda_stream);
/* enqueue one batch on cuda_stream (NULL = handle's stream).  Phase A computes
 * per-record Fletcher partials (+ codec work) and the batch aggregate. */
int32_t mtz_dev_submit(mtz_handle *h, const void *d_in, size_t in_bytes,
    const mtz_rec *d_recs, size_t nrec, void *d_out, size_t out_cap,
    void *cuda_stream);
/* aggregate (n,A,B,C,D) of the submitted batch's INPUT bytes: what a shard
 * exchanges (all-gather of 40 B) before mtz_dev_finish */
int32_t mtz_dev_aggregate(mtz_handle *h, uint64_t agg[5]);
/* phase B: verify / stamp with the running checksum that precedes the batch */
int32_t mtz_dev_finish(mtz_handle *h, const uint64_t carry_in[4],
    const uint64_t carry_out_in[4], size_t *out_bytes, uint64_t carry[4],
    uint64_t carry_out[4]);
/* stream-ordered form of the same exchange (no host round trip): the aggregate is
 * written to d_agg (5 x u64, device), the caller all-gathers it on the same CUDA
 * stream (NCCL), and hands the gathered table (world x 5 x u64, device) back; the
 * carry-in is folded from the aggregates of ranks < rank on the GPU. */
int32_t mtz_dev_aggregate_async(mtz_handle *h, void *d_agg);
int32_t mtz_dev_finish_gathered(mtz_handle *h, const void *d_all_aggs, uint32_t rank,
    const uint64_t carry_out_in[4], size_t *out_bytes, uint64_t carry[4],
    uint64_t carry_out[4]);
int32_t mtz_dev_reset(mtz_handle *h);
/* ---- the same exchange with a library-owned NCCL communicator, one process per GPU (how
 * bench.py runs under torchrun): rank 0 makes the id, the host application carries its 128
 * bytes to the other ranks (any channel), every rank calls mtz_comm_init on its handle.
 * mtz_dev_finish_exchange then does, stream-ordered and without a host round trip: all-gather
 * of the 40-byte aggregates, carry fold, verify; in the re-encoding modes the 32-byte output
 * checksum hops rank to rank (ncclRecv from rank-1, stamp chain, ncclSend to rank+1). ---- */
int32_t mtz_comm_unique_id(uint8_t id[128]);
int32_t mtz_comm_init(mtz_handle *h, const uint8_t id[128], int32_t rank, int32_t world);
/* a second handle of the same process and device rides the first one's communicator (two handles
 * alternate so that the kernels of chunk k+1 run under the exchange of chunk k) */
int32_t mtz_comm_share(mtz_handle *h, mtz_handle *owner);
/* The ranks take the stream's chunks round-robin (chunk j on rank j % world) so that the serial
 * part -- the stamp chain -- of one rank's chunk runs under the other ranks' LZ4 kernels:
 *   round_base_in   running INPUT checksum in front of this round's first chunk (NULL = zero)
 *   flags           MTZ_XCHG_FIRST: this chunk opens the stream (nothing to receive);
 *                   MTZ_XCHG_LAST: it closes it (nothing to send).  The output checksum travels
 *                   the ring rank-1 -> rank -> rank+1 (mod world).
 *   round_base_out  the base of the next round
 * One contiguous shard per rank is the special case of one round: NULL, FIRST on rank 0, LAST on
 * the last rank. */
#define MTZ_XCHG_FIRST 1u
#define MTZ_XCHG_LAST  2u
int32_t mtz_dev_finish_exchange(mtz_handle *h, const uint64_t round_base_in[4], uint32_t flags,
    size_t *out_bytes, uint64_t carry[4], uint64_t carry_out[4], uint64_t round_base_out[4]);
/* set the running checksums a slice continues from (NULL = leave) */
int32_t mtz_set_carry(mtz_handle *h, const uint64_t carry_in[4],
    const uint64_t carry_out[4]);

/* ---- kernel-level entry points: the LZ4 kernels on device-resident jobs.  The
 * stage pipeline launches exactly these; they are exported so the parity tests
 * and ncu can drive K2/K3 in isolation.  d_jobs is a device array. ---- */
/* Access contract (checked on the CPU emulator with guard pages, tests/test_emul_device_code.py):
 * decode reads exactly [src, src+src_len) and writes exactly [dst, dst+lsize); encode reads its
 * block through aligned 32-bit words, i.e. up to the 4-byte boundary at or after src+lsize and
 * down to the one at or before src, and writes only inside the lsize-byte frame slot. */
int32_t mtz_k_lz4_decode(mtz_handle *h, const void *d_src, void *d_dst,
    mtz_job *d_jobs, uint32_t njobs, void *cuda_stream);
int32_t mtz_k_lz4_encode(mtz_handle *h, const void *d_src, void *d_dst,
    mtz_job *d_jobs, uint32_t njobs, void *cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* MANATEE_GPU_H */
