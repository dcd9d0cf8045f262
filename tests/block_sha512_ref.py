"""Reference model of the block-checksum check with SHA-512 keys (MTZ_FLAG_BLOCK_SHA512) and the
stream rewrite its tests need.  Test infrastructure, on top of tests/block_sha256_ref.py (whose names
it re-exports, and so block_cksum_ref's): plain Python, numpy and hashlib over whole records.

A dataset written with checksum=sha512 carries drr_checksumtype 11.  The hash is SHA-512/256 (FIPS
180-4 5.3.6), and the 32 digest bytes are the key bytes in order: unlike a sha256 key there is no
BE_64 per word ([EXTERNAL] OpenZFS abd_checksum_sha512_native; no real checksum=sha512 stream pins
it yet).  The check classifies these records by the same table as fletcher4 keys and compares the
same bytes; only the hash differs."""
import hashlib
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from block_sha256_ref import *  # noqa: F401,F403  (records, set_key, as_sha256, trim_frames, ...)
from block_sha256_ref import (COMPRESS, DC_LZ4, DC_OFF, DECOMPRESS, FLETCHER4, FRAME_MISS, FRAME_OK,
                              LOGICAL_BAD, LOGICAL_OK, NONE, RECOMPRESS, SHA256, SKIPPED, f4, get_key,
                              records, set_key, sha256_key, trim_frames, unprop)

SHA512 = 11


def sha512_key(data):
    """the four ddk_cksum words of a SHA-512 key of `data`: the SHA-512/256 digest read as
    little-endian u64s (the digest bytes in order)"""
    return struct.unpack("<4Q", hashlib.new("sha512_256", data).digest())


def as_sha512(oracle, stream, threads=1):
    """The same stream written to a dataset with checksum=sha512: every fletcher4 key of a WRITE that
    arrives uncompressed becomes the SHA-512/256 of the bytes it covers -- the logical block, or for
    a block the key says is stored LZ4 (as_lz4_on_disk) its disk frame zero-padded to PSIZE.
    Re-stamped; composes with as_send_c and trim_frames.  `threads` hash in parallel."""
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
            return sha512_key(logical.tobytes())
        _, frame = oracle.zfs_lz4_compress(logical)
        clen = 4 + int.from_bytes(frame[:4].tobytes(), "big")
        assert clen <= psize
        return sha512_key(frame[:clen].tobytes() + bytes(psize - clen))

    if threads > 1:
        with ThreadPoolExecutor(threads) as ex:
            keys = list(ex.map(key, todo, chunksize=64))
    else:
        keys = [key(j) for j in todo]
    for (off, _, _, _), k in zip(todo, keys):
        set_key(s, off, SHA512, k)
    assert oracle.stream_restamp(s)[0] == 0
    return s


def trim_frames_to(oracle, stream, align):
    """trim_frames with the payloads rounded up to `align` bytes (a multiple of 8 that divides 512)
    instead of 8: with align=128 every frame shorter than PSIZE ends on a 128-byte block boundary,
    with align=8 most end inside one.  Re-stamped."""
    t = trim_frames(oracle, stream)
    parts = []
    for off, po, pl, typ in records(t):
        h = t[off:off + 312].copy()
        pay = t[po:po + pl]
        if typ == 3 and h[50] == DC_LZ4 and pl % align:
            pay = np.concatenate([pay, np.zeros(align - pl % align, dtype=np.uint8)])
            h[96:104] = np.frombuffer(struct.pack("<Q", pay.size), dtype=np.uint8)
        parts += [h, pay]
    s = np.ascontiguousarray(np.concatenate(parts))
    assert oracle.stream_restamp(s)[0] == 0
    return s


def block_check(inp, out, mode, sha256=False, sha512=False):
    """block_sha256_ref.block_check with MTZ_FLAG_BLOCK_SHA512: with `sha512` SHA-512 keys go through
    the same table (compared with hashlib) and counters["sha512"] counts them; without it the result
    is block_sha256_ref.block_check's plus sha512 = 0 (tests/test_block_sha512_oracle.py holds the two
    together).  The two flags are independent."""
    hashes = {FLETCHER4: lambda b: f4((0, 0, 0, 0), b)}
    if sha256:
        hashes[SHA256] = sha256_key
    if sha512:
        hashes[SHA512] = sha512_key
    ib = inp.tobytes() if isinstance(inp, np.ndarray) else bytes(inp)
    irecs = records(inp)
    orecs = records(out) if out is not None else None
    ob = out.tobytes() if out is not None else None
    verdicts, hashed = {}, {SHA256: set(), SHA512: set()}
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
        if ctype in hashes and p != 0 and not crypt and lsize == drr_lsize:
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
        if ctype in hashed:
            hashed[ctype].add(i)
        ok = data is not None and len(data) <= cover and hashes[ctype](data + bytes(cover - len(data))) == key
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
          "sha256": len(hashed[SHA256]),
          "sha512": len(hashed[SHA512])}
    return verdicts, st
