"""GpuSnapshotStage -- Python mirror of the Node ``stream.Transform`` that is
spliced into the reference's two pipes:

    zfsSend.stdout.pipe(stage).pipe(socket)     # lib/backupSender.js:179
    socket.pipe(stage).pipe(zfsRecv.stdin)      # lib/zfsClient.js:826

It is a thin object over the C ABI (include/manatee_gpu.h); every byte of work
happens in libmanatee_gpu.so on the GPU.  Node is not available in this image,
so this mirror is what the tests and ``bench.py`` drive; ``js/`` holds the Node
side a maintainer would ship (INTEGRATION.md).
"""
import ctypes as C

import numpy as np

from . import _native as N


class GpuSnapshotStage(object):
    """One stage instance == one mtz_handle == one stream (like one Transform)."""

    def __init__(self, mode="verify", device=0, ring_bytes=0, batch_bytes=0, n_slots=0,
                 out_ring_bytes=0, flags=0, devices=None, block_checksums=False, block_sha256=False,
                 block_sha512=False, block_frames=False, block_lzjb=False, block_logical=False):
        """``devices`` = CUDA ordinals of a device group: the GPUs of one box run as ONE stage,
        batch b of the stream on ``devices[b % len(devices)]`` (mtz_config.devices[]).
        ``block_checksums`` = MTZ_FLAG_BLOCK_CKSUM: every DRR_WRITE is also checked against the
        on-disk block checksum the stream carries (``block_stats()``).
        ``block_sha256`` = MTZ_FLAG_BLOCK_SHA256: the check also covers SHA-256 keys
        (checksum=sha256); only valid with ``block_checksums``, MtzError(EINVAL) otherwise.
        ``block_sha512`` = MTZ_FLAG_BLOCK_SHA512: likewise for SHA-512/256 keys (checksum=sha512),
        with or without ``block_sha256``.
        ``block_frames`` = MTZ_FLAG_BLOCK_FRAMES: in VERIFY, a block that arrives raw while its key
        covers an LZ4 frame on disk is compared with the stage's encoder frame of it instead of
        being skipped (``block_stats()["frames_encoded"]``); the other modes accept it and do not
        change.  Only valid with ``block_checksums``.
        ``block_lzjb`` = MTZ_FLAG_BLOCK_LZJB: keys over an lzjb or zle frame on disk are checked too:
        a record that arrives as that frame (VERIFY, RECOMPRESS) as it is, a raw one in VERIFY
        against the stage's lzjb / zle encoder frame of it (``block_stats()["lzjb_encoded"]``,
        ``["zle_encoded"]``).  With or without ``block_frames``; only valid with ``block_checksums``.
        ``block_logical`` = MTZ_FLAG_BLOCK_LOGICAL: COMPRESS, DECOMPRESS and RECOMPRESS also check keys
        from the logical bytes they hold, so that a transfer over the compressed wire counts what
        VERIFY counts on the raw stream: RECOMPRESS compares a raw-on-disk key of an LZ4 record with
        the decoded bytes (ECKSUM on a mismatch), with ``block_lzjb`` the three modes encode lzjb / zle
        frames of raw and LZ4 records as VERIFY does, and DECOMPRESS counts a raw record with an LZ4
        key as the frame miss the sender counted (``block_stats()["logical_checked"]``).  VERIFY
        accepts it and does not change.  Only valid with ``block_checksums``."""
        if block_checksums:
            flags |= N.FLAG_BLOCK_CKSUM
        if block_sha256:
            flags |= N.FLAG_BLOCK_SHA256
        if block_sha512:
            flags |= N.FLAG_BLOCK_SHA512
        if block_frames:
            flags |= N.FLAG_BLOCK_FRAMES
        if block_lzjb:
            flags |= N.FLAG_BLOCK_LZJB
        if block_logical:
            flags |= N.FLAG_BLOCK_LOGICAL
        self._L = N.lib()
        self._h = C.c_void_p()
        cfg = N.Config()
        cfg.struct_size = C.sizeof(N.Config)
        cfg.device = device
        if devices:
            cfg.n_devices = len(devices)
            for i, d in enumerate(devices):
                cfg.devices[i] = int(d)
        cfg.mode = N.MODE_NAMES[mode] if isinstance(mode, str) else int(mode)
        cfg.flags = flags
        cfg.ring_bytes = ring_bytes
        cfg.out_ring_bytes = out_ring_bytes
        cfg.batch_bytes = batch_bytes
        cfg.n_slots = n_slots
        rc = self._L.mtz_open(C.byref(cfg), C.byref(self._h))
        if rc != N.OK:
            msg = self._L.mtz_last_error(None)
            self._h = None
            raise N.MtzError(rc, (msg or b"").decode() or self._L.mtz_strerror(rc).decode())
        self.mode = mode

    # -- plumbing ---------------------------------------------------------
    def _check(self, rc, allow=()):
        if rc == N.OK or rc in allow:
            return rc
        msg = self._L.mtz_last_error(self._h) or b""
        raise N.MtzError(rc, msg.decode() or self._L.mtz_strerror(rc).decode())

    def close(self):
        if self._h is not None and self._h.value:
            self._L.mtz_close(self._h)
        self._h = None

    destroy = close

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def stats(self):
        st = N.Stats()
        self._check(self._L.mtz_get_stats(self._h, C.byref(st)))
        return st.as_dict()

    def block_stats(self):
        """Block-checksum counters (mtz_get_block_stats); all zero without ``block_checksums``.
        ``first_frame_miss`` is the stream index of the first frame miss, 2**64-1 if none."""
        st = N.BlockStats()
        st.struct_size = C.sizeof(N.BlockStats)
        self._check(self._L.mtz_get_block_stats(self._h, C.byref(st)))
        return st.as_dict()

    def end_checksum(self):
        out = (C.c_uint64 * 4)()
        rc = self._L.mtz_end_checksum(self._h, C.byref(out))
        if rc == N.EAGAIN:
            return None
        self._check(rc)
        return tuple(int(x) for x in out)

    # -- bulk host API ------------------------------------------------------
    def process_host(self, src, out=None):
        """Run a whole stream held in host memory through the GPU.

        ``src``/``out`` are numpy uint8 arrays (ideally from ``pinned_empty``).
        Returns the number of output bytes."""
        n_out = C.c_size_t(0)
        optr = out.ctypes.data if out is not None else None
        ocap = out.size if out is not None else 0
        self._check(self._L.mtz_process_host(self._h, src.ctypes.data, src.size, optr, ocap,
                                             C.byref(n_out)))
        return n_out.value

    # -- streaming API (Transform._write / push / _flush) -----------------
    def write(self, chunk, block=True):
        a = np.frombuffer(chunk, dtype=np.uint8) if not isinstance(chunk, np.ndarray) else chunk
        return self._check(self._L.mtz_write(self._h, a.ctypes.data, a.size, 1 if block else 0),
                           allow=(N.EAGAIN,))

    def flush(self):
        self._check(self._L.mtz_flush(self._h))

    def read(self, cap=1 << 20, block=True):
        """Returns bytes, b'' when nothing is ready (non-blocking) or None at EOF."""
        buf = np.empty(cap, dtype=np.uint8)
        got = C.c_size_t(0)
        rc = self._check(self._L.mtz_read(self._h, buf.ctypes.data, cap, C.byref(got),
                                          1 if block else 0), allow=(N.EAGAIN, N.EOF))
        if rc == N.EOF:
            return None
        return buf[:got.value].tobytes()

    def event_fd(self):
        return self._L.mtz_event_fd(self._h)

    # -- fan-out: several peers share one pass (mtz_fanout_attach) -----------
    def fanout_attach(self, peer_id):
        """Attach peer ``peer_id`` (before the first byte); returns its egress GPU ordinal."""
        rc = self._L.mtz_fanout_attach(self._h, peer_id)
        if rc < 0:
            self._check(rc)
        return rc

    def read_peer(self, peer_id, cap=1 << 20, block=True):
        buf = np.empty(cap, dtype=np.uint8)
        got = C.c_size_t(0)
        rc = self._check(self._L.mtz_read_peer(self._h, peer_id, buf.ctypes.data, cap, C.byref(got),
                                               1 if block else 0), allow=(N.EAGAIN, N.EOF))
        if rc == N.EOF:
            return None
        return buf[:got.value].tobytes()

    def peek_peer(self, peer_id):
        """(address, nbytes) of the next contiguous run in the peer's pinned ring; (0, 0) when
        nothing is ready, None at EOF."""
        p, n = C.c_void_p(), C.c_size_t()
        rc = self._check(self._L.mtz_out_peek_peer(self._h, peer_id, C.byref(p), C.byref(n)),
                         allow=(N.EAGAIN, N.EOF))
        if rc == N.EOF:
            return None
        return (p.value or 0, n.value) if rc == N.OK else (0, 0)

    def consume_peer(self, peer_id, n):
        self._check(self._L.mtz_out_consume_peer(self._h, peer_id, n))

    def cancel(self):
        """Tear the pipe down from outside: every blocked write/read returns ECANCELED."""
        if self._h is not None and self._h.value:
            self._L.mtz_cancel(self._h)

    # -- device-resident API -----------------------------------------------
    def set_carry(self, carry_in=None, carry_out=None):
        ci = (C.c_uint64 * 4)(*carry_in) if carry_in is not None else None
        co = (C.c_uint64 * 4)(*carry_out) if carry_out is not None else None
        self._check(self._L.mtz_set_carry(self._h, ci, co))

    def dev_reset(self):
        self._check(self._L.mtz_dev_reset(self._h))

    def dev_submit(self, d_in_ptr, in_bytes, d_recs_ptr, nrec, d_out_ptr=0, out_cap=0,
                   cuda_stream=0):
        self._check(self._L.mtz_dev_submit(self._h, d_in_ptr, in_bytes, d_recs_ptr, nrec,
                                           d_out_ptr or None, out_cap, cuda_stream or None))

    def dev_index(self, d_in_ptr, nbytes, d_recs_ptr, cap, cuda_stream=0):
        """GPU-side DRR parse of a resident stream -> (nrec, consumed_bytes)."""
        nrec = C.c_size_t(0)
        used = C.c_size_t(0)
        self._check(self._L.mtz_dev_index(self._h, d_in_ptr, nbytes, d_recs_ptr, cap, C.byref(nrec),
                                          C.byref(used), cuda_stream or None))
        return nrec.value, used.value

    def dev_aggregate(self):
        agg = (C.c_uint64 * 5)()
        self._check(self._L.mtz_dev_aggregate(self._h, C.byref(agg)))
        return tuple(int(x) for x in agg)

    def dev_aggregate_async(self, d_agg_ptr):
        self._check(self._L.mtz_dev_aggregate_async(self._h, d_agg_ptr))

    def dev_finish_gathered(self, d_all_aggs_ptr, rank, carry_out_in=None):
        ob = C.c_size_t(0)
        c1 = (C.c_uint64 * 4)()
        c2 = (C.c_uint64 * 4)()
        co = (C.c_uint64 * 4)(*carry_out_in) if carry_out_in is not None else None
        self._check(self._L.mtz_dev_finish_gathered(self._h, d_all_aggs_ptr, rank, co, C.byref(ob),
                                                    C.byref(c1), C.byref(c2)))
        return ob.value, tuple(int(x) for x in c1), tuple(int(x) for x in c2)

    def comm_init(self, unique_id, rank, world):
        """Library-owned NCCL communicator for the one-process-per-GPU shard form."""
        buf = (C.c_uint8 * 128).from_buffer_copy(bytes(unique_id))
        self._check(self._L.mtz_comm_init(self._h, buf, rank, world))

    def comm_share(self, owner):
        """Ride the communicator of another handle of this process (same device)."""
        self._check(self._L.mtz_comm_share(self._h, owner._h))

    def dev_finish_exchange(self, round_base=None, flags=None, rank=None, world=None):
        """Finish the submitted chunk with the library-owned exchange.  Default flags = one
        contiguous shard per rank (FIRST on rank 0, LAST on the last rank).  Returns
        (out_bytes, carry, carry_out, round_base_out)."""
        if flags is None:
            flags = (N.XCHG_FIRST if rank in (None, 0) else 0) | \
                (N.XCHG_LAST if (rank is None or world is None or rank == world - 1) else 0)
        ob = C.c_size_t(0)
        c1 = (C.c_uint64 * 4)()
        c2 = (C.c_uint64 * 4)()
        nb = (C.c_uint64 * 4)()
        bi = (C.c_uint64 * 4)(*round_base) if round_base is not None else None
        self._check(self._L.mtz_dev_finish_exchange(self._h, bi, flags, C.byref(ob), C.byref(c1), C.byref(c2),
                                                    C.byref(nb)))
        return ob.value, tuple(int(x) for x in c1), tuple(int(x) for x in c2), tuple(int(x) for x in nb)

    def dev_finish(self, carry_in=None, carry_out_in=None):
        ob = C.c_size_t(0)
        c1 = (C.c_uint64 * 4)()
        c2 = (C.c_uint64 * 4)()
        ci = (C.c_uint64 * 4)(*carry_in) if carry_in is not None else None
        co = (C.c_uint64 * 4)(*carry_out_in) if carry_out_in is not None else None
        self._check(self._L.mtz_dev_finish(self._h, ci, co, C.byref(ob), C.byref(c1), C.byref(c2)))
        return ob.value, tuple(int(x) for x in c1), tuple(int(x) for x in c2)


def comm_unique_id():
    """128 bytes to carry from rank 0 to the other ranks (mtz_comm_unique_id)."""
    L = N.lib()
    buf = (C.c_uint8 * 128)()
    rc = L.mtz_comm_unique_id(buf)
    if rc != N.OK:
        raise N.MtzError(rc, "mtz_comm_unique_id")
    return bytes(buf)


def index_host(stream):
    """Host-side DRR parse: numpy structured array of mtz_rec for whole records."""
    L = N.lib()
    a = stream
    nrec = C.c_size_t(0)
    used = C.c_size_t(0)
    rc = L.mtz_index_host(a.ctypes.data, a.size, None, 0, C.byref(nrec), C.byref(used))
    if rc != N.OK:
        raise N.MtzError(rc, L.mtz_strerror(rc).decode())
    recs = np.zeros(nrec.value, dtype=REC_DTYPE)
    rc = L.mtz_index_host(a.ctypes.data, a.size, recs.ctypes.data, recs.size, C.byref(nrec),
                          C.byref(used))
    if rc != N.OK:
        raise N.MtzError(rc, L.mtz_strerror(rc).decode())
    return recs, used.value


REC_DTYPE = np.dtype([("off", "<u8"), ("payload", "<u4"), ("type", "<u4"), ("lsize", "<u4"),
                      ("comp", "<u4"), ("resv", "<u8")])


class PinnedBuffer(object):
    """numpy view over cudaHostAlloc memory (mtz_host_alloc / mtz_host_free)."""

    def __init__(self, nbytes):
        self._L = N.lib()
        p = C.c_void_p()
        rc = self._L.mtz_host_alloc(nbytes, C.byref(p))
        if rc != N.OK:
            raise N.MtzError(rc, "mtz_host_alloc(%d)" % nbytes)
        self._p = p
        self.array = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p.value))

    def free(self):
        if self._p is not None:
            self.array = None
            self._L.mtz_host_free(self._p)
            self._p = None
