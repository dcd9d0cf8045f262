"""Reference model of the block-checksum check with MTZ_FLAG_BLOCK_LOGICAL.  Test infrastructure, on
top of tests/block_lzjb_ref.py (whose names it re-exports): plain Python, numpy, hashlib, the oracle.

With the flag COMPRESS, DECOMPRESS and RECOMPRESS also check keys from the logical bytes they hold:
the input payload of a record that arrives raw, the decoded payload of one that arrives LZ4.
  1. a raw-on-disk key of a record that arrives LZ4 in RECOMPRESS is compared with them (DECOMPRESS
     already compares it with its output);
  2. with MTZ_FLAG_BLOCK_LZJB, an lzjb / zle key of a record that arrives raw, or LZ4 where the mode
     decodes it (DECOMPRESS, RECOMPRESS; not COMPRESS), is compared with the declared encoder's frame of
     them, as VERIFY compares a raw record;
  3. an LZ4 key of a record that arrives raw in DECOMPRESS is the frame miss COMPRESS counted for it
     when its encoder stored the block raw.
So a stream counts the same in VERIFY on its raw form and in every stage of the compressed wire."""
import struct

import numpy as np

from block_lzjb_ref import *  # noqa: F401,F403  (records, set_key, as_on_disk, block_check_lzjb, ...)
from block_lzjb_ref import (COMPRESS, DC_LZ4, DC_LZJB, DC_OFF, DC_ZLE, DECOMPRESS, FLETCHER4, FRAME_MISS,
                            FRAME_OK, LOGICAL_BAD, LOGICAL_OK, RECOMPRESS, SHA256, SHA512, SKIPPED, VERIFY,
                            as_on_disk, block_check_lzjb, disk_frame, encoder_frame, f4, get_key, prop,
                            records, set_key, sha256_key, sha512_key, unprop)

DC_ZSTD = 16
CKSUM_SKEIN = 12            # a salted hash: never checkable
COUNTERS = ("logical_ok", "frame_ok", "frame_miss", "skipped", "first_frame_miss", "sha256", "sha512",
            "lzjb_encoded", "zle_encoded")
FLAGS = ("sha256", "sha512", "frames", "lzjb")


def block_check_logical(oracle, inp, mode, out=None, frames=False, lzjb=False, sha256=False, sha512=False,
                        logical=True):
    """The verdicts and counters of the block check in `mode` on the plain stream `inp` (`out` = the
    stage's plain output, None in VERIFY) with MTZ_FLAG_BLOCK_LOGICAL = `logical`: block_check_lzjb's
    with the records the flag adds.  counters["logical_checked"] counts them."""
    verdicts, st = block_check_lzjb(oracle, inp, mode=mode, frames=frames, lzjb=lzjb, sha256=sha256,
                                    sha512=sha512, out=out)
    st["logical_checked"] = 0
    if not logical or mode not in (COMPRESS, DECOMPRESS, RECOMPRESS):
        return verdicts, st
    hashes = {FLETCHER4: lambda x: f4((0, 0, 0, 0), x)}
    if sha256:
        hashes[SHA256] = sha256_key
    if sha512:
        hashes[SHA512] = sha512_key
    b = inp.tobytes() if isinstance(inp, np.ndarray) else bytes(inp)
    for i, (off, po, pl, t) in enumerate(records(inp)):
        if t != 3 or verdicts[i] != SKIPPED:
            continue
        h = b[off:off + 312]
        ctype, arrive = h[48], h[50]
        key = struct.unpack_from("<4Q", h, 56)
        p = int.from_bytes(h[88:96], "little")
        lsize, psize, dc, crypt = unprop(p)
        drr_lsize = int.from_bytes(h[32:40], "little")
        if ctype not in hashes or p == 0 or crypt or lsize != drr_lsize or arrive not in (0, DC_LZ4):
            continue
        if arrive == DC_LZ4 and mode == COMPRESS:
            continue                                 # COMPRESS decodes nothing: no logical bytes of an LZ4 record

        def logical_bytes():
            if arrive == 0:
                return b[po:po + pl]
            rc, d = oracle.zfs_lz4_decompress(np.frombuffer(b[po:po + pl], dtype=np.uint8), lsize)
            assert rc == 0
            return d.tobytes()

        if dc in (0, DC_OFF) and psize == lsize and arrive == DC_LZ4 and mode == RECOMPRESS:
            ok = hashes[ctype](logical_bytes()) == key
            verdicts[i] = LOGICAL_OK if ok else LOGICAL_BAD
            st["logical_ok"] += ok
            if not ok:
                st["first_bad"] = min(st["first_bad"], i)
        elif dc in (DC_LZJB, DC_ZLE) and lzjb:
            fr = encoder_frame(dc, logical_bytes())
            st["lzjb_encoded" if dc == DC_LZJB else "zle_encoded"] += 1
            ok = fr is not None and len(fr) <= psize and hashes[ctype](fr + bytes(psize - len(fr))) == key
            verdicts[i] = FRAME_OK if ok else FRAME_MISS
        elif dc == DC_LZ4 and arrive == 0 and mode == DECOMPRESS:
            verdicts[i] = FRAME_MISS
        else:
            continue
        st["skipped"] -= 1
        st["logical_checked"] += 1
        if verdicts[i] in (FRAME_OK, FRAME_MISS):
            st[verdicts[i]] += 1
            if verdicts[i] == FRAME_MISS:
                st["first_frame_miss"] = min(st["first_frame_miss"], i)
        if ctype in (SHA256, SHA512):
            st["sha256" if ctype == SHA256 else "sha512"] += 1
    return verdicts, st


def mixed_keys_stream(oracle, n=40, recsize=8192, seed=0):
    """A raw stream (`zfs send` without -c) whose records carry a seeded mix of keys: on-disk lzjb, zle,
    LZ4 and raw; fletcher4, sha256 and sha512; and every ninth or so one the stage cannot check (zstd on
    disk, encrypted, a salted hash).  pg-page records with incompressible and all-zero ones mixed in, so
    some compressed-on-disk picks end up stored raw, and some of those carry an LZ4 key that no frame of
    the stage can match.  Returns (stream, {record index: on-disk compression
    of the checkable ones})."""
    from test_gpu_codec import _mixed_stream
    rng = np.random.default_rng(seed)
    picks = rng.integers(0, 4, 2 * n + 8)
    s, dcs = as_on_disk(oracle, _mixed_stream(oracle, n=n, recsize=recsize), 9,
                        lambda i: (DC_LZJB, DC_ZLE, DC_LZ4, DC_OFF)[picks[i]])
    for i, (off, po, pl, t) in enumerate(records(s)):
        if i not in dcs:
            continue
        lsize, psize, dc, _ = unprop(get_key(s, off)[2])
        logical = s[po:po + pl]
        data = logical.tobytes() if dcs[i] == DC_OFF else disk_frame(oracle, logical, 9, dc).tobytes()
        if dcs[i] == DC_OFF and picks[i] != 3 and i % 2 == 0 and lsize > 512:
            # a block no declared encoder shrinks, keyed as if another LZ4 encoder had: a frame miss wherever
            # it is checked, and on the compressed wire a record that travels raw under an LZ4 key
            set_key(s, off, ddk_prop=prop(lsize, lsize - 512, DC_LZ4))
            dcs[i] = DC_LZ4
        how = int(rng.integers(0, 9))
        if how in (1, 2):
            set_key(s, off, SHA256, sha256_key(data))
        elif how in (3, 4):
            set_key(s, off, SHA512, sha512_key(data))
        elif how == 5:
            kind = int(rng.integers(0, 3))
            if kind == 0:
                set_key(s, off, ddk_prop=prop(lsize, psize, DC_ZSTD))
            elif kind == 1:
                set_key(s, off, ddk_prop=prop(lsize, psize, dc, crypt=1))
            else:
                set_key(s, off, ctype=CKSUM_SKEIN)
            del dcs[i]
    assert oracle.stream_restamp(s)[0] == 0
    return s, dcs


def send_c_form(oracle, x):
    """the compressed form of a raw stream the RECOMPRESS tests feed the stage: every record the oracle's
    encoder can store as an LZ4 frame travels as one, whatever its key says"""
    rc, c, _ = oracle.stream_compress_plain(x)
    assert rc == 0
    return np.ascontiguousarray(c)


def four_ways(oracle, x, **flags):
    """the model's counters of the four stages of the invariant on the raw stream `x`, `flags` a subset of
    FLAGS: VERIFY on x, COMPRESS on x, DECOMPRESS on COMPRESS(x), RECOMPRESS on the send-c form"""
    c = send_c_form(oracle, x)
    rc, d, _ = oracle.stream_decompress(oracle.stream_compress(x)[1])
    rc2, r, _ = oracle.stream_recompress(c)
    assert rc == 0 and rc2 == 0 and np.array_equal(d, x)
    return {"verify": block_check_logical(oracle, x, VERIFY, None, **flags),
            "compress": block_check_logical(oracle, x, COMPRESS, c, **flags),
            "decompress": block_check_logical(oracle, c, DECOMPRESS, x, **flags),
            "recompress": block_check_logical(oracle, c, RECOMPRESS, r, **flags)}
