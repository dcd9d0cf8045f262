"""Reference model of the block-checksum check with SHA-256 keys (MTZ_FLAG_BLOCK_SHA256) and the
stream rewrites its tests need.  Test infrastructure, on top of tests/block_cksum_ref.py (whose
names it re-exports): plain Python, numpy and hashlib over whole records.

A dataset written with checksum=sha256 carries drr_checksumtype 8; the key words are the FIPS 180-4
digest's big-endian u64s ([EXTERNAL] OpenZFS zio_checksum_SHA256), stored as native little-endian
words like every other key.  The check classifies these records by the same table as fletcher4 keys
and compares the same bytes; only the hash differs."""
import hashlib
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from block_cksum_ref import *  # noqa: F401,F403  (records, prop, set_key, as_lz4_on_disk, as_send_c, ...)
from block_cksum_ref import (COMPRESS, DC_LZ4, DC_OFF, DECOMPRESS, FLETCHER4, FRAME_MISS, FRAME_OK,
                             LOGICAL_BAD, LOGICAL_OK, NONE, RECOMPRESS, SHA256, SKIPPED, f4, get_key,
                             records, set_key, unprop)


def sha256_key(data):
    """the four ddk_cksum words of a SHA-256 key of `data`: BE_64 of the digest's 8-byte groups"""
    return struct.unpack(">4Q", hashlib.sha256(data).digest())


def as_sha256(oracle, stream, threads=1):
    """The same stream written to a dataset with checksum=sha256: every fletcher4 key of a WRITE that
    arrives uncompressed becomes the SHA-256 of the bytes it covers -- the logical block, or for a
    block the key says is stored LZ4 (as_lz4_on_disk) its disk frame zero-padded to PSIZE.
    Re-stamped; composes with as_send_c.  `threads` hash in parallel (hashlib releases the GIL)."""
    s = np.array(stream, dtype=np.uint8, copy=True)
    todo = []
    for off, po, pl, t in records(s):
        if t != 3 or s[off + 50] != 0 or s[off + 48] != FLETCHER4:
            continue
        _, _, p = get_key(s, off)
        todo.append((off, po, pl, unprop(p)))

    def key(job):
        off, po, pl, (lsize, psize, dc, _) = job
        logical = s[po:po + pl]
        if dc != DC_LZ4:
            return sha256_key(logical.tobytes())
        _, frame = oracle.zfs_lz4_compress(logical)
        clen = 4 + int.from_bytes(frame[:4].tobytes(), "big")
        assert clen <= psize
        return sha256_key(frame[:clen].tobytes() + bytes(psize - clen))

    if threads > 1:
        with ThreadPoolExecutor(threads) as ex:
            keys = list(ex.map(key, todo, chunksize=64))
    else:
        keys = [key(j) for j in todo]
    for (off, _, _, _), k in zip(todo, keys):
        set_key(s, off, SHA256, k)
    assert oracle.stream_restamp(s)[0] == 0
    return s


def trim_frames(oracle, stream):
    """A `send -c` stream whose LZ4 payloads stop at the frame's end rounded up to 8 bytes instead of
    PSIZE (compressed_size follows; the keys, which cover PSIZE, stay): the bytes at hand are shorter
    than what the key covers and end anywhere in a 64-byte block.  Re-stamped."""
    parts = []
    b = np.asarray(stream, dtype=np.uint8)
    for off, po, pl, t in records(b):
        h = b[off:off + 312].copy()
        pay = b[po:po + pl]
        if t == 3 and h[50] == DC_LZ4:
            n = (4 + int.from_bytes(pay[:4].tobytes(), "big") + 7) & ~7
            if n < pl:
                pay = pay[:n]
                h[96:104] = np.frombuffer(struct.pack("<Q", n), dtype=np.uint8)
        parts += [h, pay]
    s = np.ascontiguousarray(np.concatenate(parts))
    assert oracle.stream_restamp(s)[0] == 0
    return s


def block_check(inp, out, mode, sha256=False):
    """block_cksum_ref.block_check with MTZ_FLAG_BLOCK_SHA256: with `sha256` SHA-256 keys go through
    the same table (compared with hashlib) and counters["sha256"] counts them; without it the result
    is block_cksum_ref.block_check's (tests/test_block_sha256_oracle.py holds the two together)."""
    ib = inp.tobytes() if isinstance(inp, np.ndarray) else bytes(inp)
    irecs = records(inp)
    orecs = records(out) if out is not None else None
    ob = out.tobytes() if out is not None else None
    verdicts, hashed = {}, set()
    for i, (off, po, pl, t) in enumerate(irecs):
        if t != 3:
            continue
        h = ib[off:off + 312]
        ctype = h[48]
        key = struct.unpack_from("<4Q", h, 56)
        p = struct.unpack_from("<Q", h, 88)[0]
        lsize, psize, dc, crypt = unprop(p)
        arrive = h[50]
        drr_lsize = struct.unpack_from("<Q", h, 32)[0]
        src = None                                   # (bytes at hand, what they are)
        if (ctype == FLETCHER4 or (sha256 and ctype == SHA256)) and p != 0 and not crypt and lsize == drr_lsize:
            if dc in (0, DC_OFF) and psize == lsize:
                if arrive == 0:
                    src = (ib[po:po + pl], "logical")
                elif arrive == DC_LZ4 and mode == DECOMPRESS:
                    _, opo, opl, _ = orecs[i]
                    src = (ob[opo:opo + opl], "logical")
            elif dc == DC_LZ4:
                if arrive == DC_LZ4:
                    src = (ib[po:po + pl], "frame")
                elif arrive == 0 and mode in (COMPRESS, RECOMPRESS):
                    ooff, opo, opl, _ = orecs[i]
                    # the stage stored the block raw where ZFS stored a frame: no frame to compare
                    src = (ob[opo:opo + opl] if ob[ooff + 50] == DC_LZ4 else None, "frame")
        if src is None:
            verdicts[i] = SKIPPED
            continue
        data, what = src
        cover = lsize if what == "logical" else psize
        if ctype == SHA256:
            hashed.add(i)
            digest = sha256_key
        else:
            def digest(b):
                return f4((0, 0, 0, 0), b)
        ok = data is not None and len(data) <= cover and digest(data + bytes(cover - len(data))) == key
        if what == "logical":
            verdicts[i] = LOGICAL_OK if ok else LOGICAL_BAD
        else:
            verdicts[i] = FRAME_OK if ok else FRAME_MISS
    v = list(verdicts.items())
    st = {"logical_ok": sum(1 for _, x in v if x == LOGICAL_OK),
          "frame_ok": sum(1 for _, x in v if x == FRAME_OK),
          "frame_miss": sum(1 for _, x in v if x == FRAME_MISS),
          "skipped": sum(1 for _, x in v if x == SKIPPED),
          "first_frame_miss": min([i for i, x in v if x == FRAME_MISS], default=NONE),
          "first_bad": min([i for i, x in v if x == LOGICAL_BAD], default=NONE),
          "sha256": len(hashed)}
    return verdicts, st

