"""Reference model of the block-checksum check in VERIFY with MTZ_FLAG_BLOCK_FRAMES.  Test
infrastructure, on top of tests/block_sha512_ref.py (whose names it re-exports, and so those of
block_sha256_ref and block_cksum_ref): plain Python, numpy, hashlib and the oracle's LZ4 encoder.

A block ZFS stored LZ4 has a key over its disk frame.  When it arrives raw (`zfs send` without -c),
VERIFY alone skips it; with the flag the stage encodes it with the declared encoder and compares
that frame by the rules COMPRESS applies to its own output.  So the verdicts of VERIFY + frames on a
stream are those of COMPRESS on it: block_check(inp, COMPRESS(inp), COMPRESS).  The model below
(block_check_frames) computes them record by record, which also covers a stream COMPRESS refuses (an already compressed
one); tests/test_block_frames_oracle.py holds it to the COMPRESS composition."""
import struct

import numpy as np

from block_sha512_ref import *  # noqa: F401,F403  (records, set_key, as_lz4_on_disk, as_sha512, ...)
from block_sha512_ref import (DC_LZ4, FLETCHER4, FRAME_MISS, FRAME_OK, SHA256, SHA512, SKIPPED, VERIFY,
                              f4, records, sha256_key, sha512_key, unprop)
import block_sha512_ref as _S


def encoder_frame(oracle, logical):
    """What the stage's encoder stores for `logical`: the frame zero-padded to its 512-byte PSIZE,
    or None when it stores the block raw (the oracle's zfs_lz4_compress, the declared encoder)"""
    ps, frame = oracle.zfs_lz4_compress(logical)
    if frame is None:
        return None
    clen = 4 + int.from_bytes(frame[:4].tobytes(), "big")
    return frame[:clen].tobytes() + bytes(ps - clen)


def block_check_frames(oracle, inp, sha256=False, sha512=False):
    """VERIFY + MTZ_FLAG_BLOCK_FRAMES: block_sha512_ref.block_check(inp, None, VERIFY, ...) with every
    record that arrives raw while its checkable key covers an LZ4 frame compared with
    encoder_frame() instead of being skipped.  counters["frames_encoded"] counts those records."""
    verdicts, st = _S.block_check(inp, None, VERIFY, sha256=sha256, sha512=sha512)
    hashes = {FLETCHER4: lambda b: f4((0, 0, 0, 0), b)}
    if sha256:
        hashes[SHA256] = sha256_key
    if sha512:
        hashes[SHA512] = sha512_key
    b = inp.tobytes() if isinstance(inp, np.ndarray) else bytes(inp)
    frames = 0
    for i, (off, po, pl, t) in enumerate(records(inp)):
        if t != 3 or verdicts[i] != SKIPPED:
            continue
        h = b[off:off + 312]
        ctype, arrive = h[48], h[50]
        key = struct.unpack_from("<4Q", h, 56)
        p = int.from_bytes(h[88:96], "little")
        lsize, psize, dc, crypt = unprop(p)
        drr_lsize = int.from_bytes(h[32:40], "little")
        if ctype not in hashes or p == 0 or crypt or lsize != drr_lsize or dc != DC_LZ4 or arrive != 0:
            continue
        frames += 1
        fr = encoder_frame(oracle, np.frombuffer(b[po:po + pl], dtype=np.uint8))
        ok = fr is not None and len(fr) <= psize and hashes[ctype](fr + bytes(psize - len(fr))) == key
        verdicts[i] = FRAME_OK if ok else FRAME_MISS
        st["skipped"] -= 1
        st["frame_ok" if ok else "frame_miss"] += 1
        if not ok:
            st["first_frame_miss"] = min(st["first_frame_miss"], i)
        if ctype in (SHA256, SHA512):
            st["sha256" if ctype == SHA256 else "sha512"] += 1
    st["frames_encoded"] = frames
    return verdicts, st
