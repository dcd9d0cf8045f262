"""Reference model of the block-checksum check with MTZ_FLAG_BLOCK_LZJB, and the lzjb / zle encoders
it rests on.  Test infrastructure, on top of tests/block_frames_ref.py (whose names it re-exports):
plain Python, numpy, hashlib, the oracle and tests/lzjb_zfs.c.

A block ZFS stored with compression=lzjb (on-disk compression 3) or zle (14) has a key over that
frame, zero-padded to PSIZE.  With the flag the stage compares a record that arrives as that frame
(`zfs send -c`, VERIFY and RECOMPRESS) as it is, and in VERIFY encodes a record that arrives raw with
the declared encoder and compares the frame by the rules of the LZ4 frames (block_frames_ref).

Two restatements of ZFS's encoders live here: tests/lzjb_zfs.c, ZFS's C code on real pointers
(`phase` = the source buffer's address mod 1024, which lzjb's output depends on), and an independent
pure-Python one (py_lzjb_compress, py_zle_compress) that models phase 0 the way the GPU does: a
table entry is the position's low 16 bits, 0 for "never written"."""
import ctypes as C
import hashlib
import os
import shutil
import struct
import subprocess
import tempfile

import numpy as np

from block_frames_ref import *  # noqa: F401,F403  (records, set_key, as_lz4_on_disk, block_check_frames, ...)
from block_frames_ref import (DC_LZ4, DC_OFF, FEAT_COMPRESSED, FEAT_LZ4, FLETCHER4, FRAME_MISS, FRAME_OK,
                              SHA256, SHA512, SKIPPED, VERIFY, RECOMPRESS, f4, get_key, prop, records,
                              set_key, sha256_key, sha512_key, unprop)
import block_frames_ref as _F

DC_LZJB, DC_ZLE = 3, 14
ZLE_N = 64
_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "lzjb_zfs.c")
_lib = None


def lib():
    """tests/lzjb_zfs.c as a shared library, compiled once into a temporary directory keyed by the
    source's hash (the tree may be read-only)"""
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), "mtz_lzjb_oracle_%d" % os.getuid())
        so = os.path.join(d, "lzjb_zfs_%s.so" % hashlib.sha256(src).hexdigest()[:16])
        if not os.path.exists(so):
            os.makedirs(d, exist_ok=True)
            tmp = tempfile.mkdtemp(dir=d)
            out = os.path.join(tmp, "lib.so")
            subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=gnu11", "-Wall", "-shared", "-fPIC",
                                   "-o", out, _SRC])
            os.replace(out, so)
            shutil.rmtree(tmp, ignore_errors=True)
        L = C.CDLL(so)
        vp, sz = C.c_void_p, C.c_size_t
        L.orc_zfs_lzjb_compress.argtypes = [vp, sz, vp, C.POINTER(sz), C.c_uint]
        L.orc_zfs_lzjb_compress.restype = sz
        L.orc_zfs_zle_compress.argtypes = [vp, sz, vp, C.POINTER(sz)]
        L.orc_zfs_zle_compress.restype = sz
        for f in (L.orc_lzjb_decompress, L.orc_zle_decompress):
            f.argtypes = [vp, sz, vp, sz]
            f.restype = C.c_int
        _lib = L
    return _lib


def _cbuf(b):
    b = bytes(b)
    return C.create_string_buffer(b, len(b)), len(b)


def zfs_lzjb_compress(src, phase=0):
    """the C restatement driven as zio_compress_data: (psize, frame padded to psize) or (len, None)
    when ZFS stores the block raw, plus the encoder's own result: ((psize, frame), c_len)"""
    s, n = _cbuf(src)
    d = C.create_string_buffer(n)
    c = C.c_size_t()
    ps = lib().orc_zfs_lzjb_compress(s, n, d, C.byref(c), phase)
    return (ps, None if ps >= n else d.raw[:ps]), c.value


def zfs_zle_compress(src):
    s, n = _cbuf(src)
    d = C.create_string_buffer(n)
    c = C.c_size_t()
    ps = lib().orc_zfs_zle_compress(s, n, d, C.byref(c))
    return (ps, None if ps >= n else d.raw[:ps]), c.value


def zfs_lzjb_decompress(frame, lsize):
    s, n = _cbuf(frame)
    d = C.create_string_buffer(lsize)
    rc = lib().orc_lzjb_decompress(s, n, d, lsize)
    return None if rc != 0 else d.raw[:lsize]


def zfs_zle_decompress(frame, lsize):
    s, n = _cbuf(frame)
    d = C.create_string_buffer(lsize)
    rc = lib().orc_zle_decompress(s, n, d, lsize)
    return None if rc != 0 else d.raw[:lsize]


# ---- the independent pure-Python restatement (phase 0) ----------------------------------------------

def py_lzjb_compress(src):
    """lzjb_compress(src, dst, s_len, d_len = s_len - s_len/8) at phase 0: (c_len, frame bytes), c_len =
    s_len when the encoder gives up"""
    b = bytes(src)
    s_len = len(b)
    d_len = s_len - (s_len >> 3)
    tab = [0] * 1024
    out = bytearray()
    cm_pos, cm_bit, p = -1, 0x80, 0
    while p < s_len:
        cm_bit <<= 1
        if cm_bit == 0x100:
            if len(out) >= d_len - 1 - 16:
                return s_len, None
            cm_bit, cm_pos = 1, len(out)
            out.append(0)
        if p > s_len - 66:
            out.append(b[p])
            p += 1
            continue
        h = (b[p] << 16) + (b[p + 1] << 8) + b[p + 2]
        h += h >> 9
        h += h >> 5
        h &= 1023
        off = (p - tab[h]) & 1023
        tab[h] = p & 0xffff
        c = p - off
        if c >= 0 and c != p and b[c:c + 3] == b[p:p + 3]:
            out[cm_pos] |= cm_bit
            m = 3
            while m < 66 and b[p + m] == b[c + m]:
                m += 1
            out += bytes((((m - 3) << 2) | (off >> 8), off & 0xff))
            p += m
        else:
            out.append(b[p])
            p += 1
    return len(out), bytes(out)


def py_lzjb_decompress(frame, lsize):
    f, out, i, cm, bit = bytes(frame), bytearray(), 0, 0, 0x80
    while len(out) < lsize:
        bit <<= 1
        if bit == 0x100:
            cm, bit = f[i], 1
            i += 1
        if cm & bit:
            m = (f[i] >> 2) + 3
            off = ((f[i] << 8) | f[i + 1]) & 1023
            i += 2
            c = len(out) - off
            if c < 0:
                return None
            for _ in range(min(m, lsize - len(out))):
                out.append(out[c])
                c += 1
        else:
            out.append(f[i])
            i += 1
    return bytes(out)


def py_zle_compress(src):
    """zle_compress(src, dst, s_len, d_len = s_len - s_len/8, 64): (c_len, frame), c_len = s_len when the
    encoder gives up or does not consume the whole source"""
    b = bytes(src)
    s_len = len(b)
    d_len = s_len - (s_len >> 3)
    out = bytearray()
    p = 0
    while p < s_len and len(out) < d_len - 1:
        first = p
        if b[p] == 0:
            lim = min(p + 256 - ZLE_N, s_len)
            while p < lim and b[p] == 0:
                p += 1
            out.append(p - first - 1 + ZLE_N)
        else:
            if d_len - (len(out) + 1) < ZLE_N:
                break
            lim = min(p + ZLE_N, s_len)
            while p < lim - 1 and (b[p] | b[p + 1]):
                p += 1
            if b[p]:
                p += 1
            out.append(p - first - 1)
            out += b[first:p]
    if p != s_len:
        return s_len, None
    return len(out), bytes(out)


def py_zle_decompress(frame, lsize):
    f, out, i = bytes(frame), bytearray(), 0
    while i < len(f) and len(out) < lsize:
        n = 1 + f[i]
        i += 1
        if n <= ZLE_N:
            if i + n > len(f) or len(out) + n > lsize:
                return None
            out += f[i:i + n]
            i += n
        else:
            n -= ZLE_N
            if len(out) + n > lsize:
                return None
            out += bytes(n)
    return bytes(out) if len(out) == lsize else None


def zio_rule(c_len, frame, s_len):
    """zio_compress_data: (psize, frame zero-padded to psize), or (s_len, None) = stored raw"""
    if frame is None or c_len > s_len - (s_len >> 3):
        return s_len, None
    ps = (c_len + 511) & ~511
    if ps >= s_len:
        return s_len, None
    return ps, frame[:c_len] + bytes(ps - c_len)


# ---- streams and the model of the check --------------------------------------------------------------

def encoder_frame(codec, logical, phase=0):
    """what the stage's encoder of `codec` (DC_LZJB / DC_ZLE) stores for `logical`: the frame zero-padded
    to its 512-byte PSIZE, or None when it stores the block raw (the C restatement at phase 0)"""
    (_, fr), _ = zfs_lzjb_compress(logical, phase) if codec == DC_LZJB else zfs_zle_compress(logical)
    return fr


def disk_frame(oracle, logical, ashift, codec):
    """what ZFS with compression=`codec` (DC_LZ4, DC_LZJB or DC_ZLE) writes for `logical` at this
    ashift: the frame zero-padded to PSIZE, or None when it stores the block raw"""
    if codec == DC_LZ4:
        return _F.disk_frame(oracle, logical, ashift)
    fr = encoder_frame(codec, logical)
    if fr is None:
        return None
    # the 512-padded frame rounded up to the ashift: the same bytes zero-extended
    psize = -(-len(fr) // (1 << ashift)) << ashift
    if psize >= len(logical):
        return None
    return np.frombuffer(fr + bytes(psize - len(fr)), dtype=np.uint8)


def as_on_disk(oracle, stream, ashift=9, codec=DC_LZJB):
    """A raw stream whose keys say "written by ZFS with compression=codec at this ashift", `codec` one of
    DC_LZ4 / DC_LZJB / DC_ZLE / DC_OFF or a function of the record index that returns one: each block's
    key is the Fletcher-4 of its disk frame, or of its logical bytes where ZFS would have stored it raw.
    Re-stamped.  Returns (stream, {record index: on-disk compression})."""
    pick = codec if callable(codec) else (lambda i: codec)
    s = np.array(stream, dtype=np.uint8, copy=True)
    dcs = {}
    for i, (off, po, pl, t) in enumerate(records(s)):
        if t != 3 or s[off + 50] != 0:
            continue
        logical = s[po:po + pl]
        dc = pick(i)
        fr = None if dc == DC_OFF else disk_frame(oracle, logical, ashift, dc)
        if fr is None:
            set_key(s, off, FLETCHER4, f4((0, 0, 0, 0), logical.tobytes()), prop(pl, pl, DC_OFF))
            dcs[i] = DC_OFF
        else:
            set_key(s, off, FLETCHER4, f4((0, 0, 0, 0), fr.tobytes()), prop(pl, fr.size, dc))
            dcs[i] = dc
    assert oracle.stream_restamp(s)[0] == 0
    return s, dcs


def as_lzjb_on_disk(oracle, stream, ashift=9, codec=DC_LZJB):
    return as_on_disk(oracle, stream, ashift, codec)


def mixed_codecs(i):
    """lzjb, zle, lz4 and (unchanged: logical) keys in turn"""
    return (DC_LZJB, DC_ZLE, DC_LZ4, DC_LZJB, DC_OFF)[i % 5]


def as_send_c(oracle, stream, ashift=9):
    """The `zfs send -c` form of an as_on_disk() stream: every block stored compressed on disk travels
    as its disk frame (payload = the frame zero-padded to PSIZE, compression = the on-disk one,
    compressed_size = PSIZE), the BEGIN announces compressed records.  Re-stamped."""
    parts = []
    b = np.asarray(stream, dtype=np.uint8)
    for off, po, pl, t in records(b):
        h = b[off:off + 312].copy()
        pay = b[po:po + pl]
        if t == 0:
            vi = struct.unpack_from("<Q", h.tobytes(), 16)[0] | ((FEAT_COMPRESSED | FEAT_LZ4) << 2)
            h[16:24] = np.frombuffer(struct.pack("<Q", vi), dtype=np.uint8)
        if t == 3 and h[50] == 0:
            _, _, p = get_key(h, 0)
            lsize, psize, dc, _ = unprop(p)
            if dc in (DC_LZ4, DC_LZJB, DC_ZLE):
                fr = disk_frame(oracle, pay, ashift, dc)
                assert fr is not None and fr.size == psize
                h[50] = dc
                h[96:104] = np.frombuffer(struct.pack("<Q", psize), dtype=np.uint8)
                pay = fr
        parts += [h, pay]
    s = np.ascontiguousarray(np.concatenate(parts))
    assert oracle.stream_restamp(s)[0] == 0
    return s


def as_sha(oracle, stream, name):
    """every fletcher4 key of a WRITE that arrives raw becomes the SHA-256 (name "sha256") or
    SHA-512/256 ("sha512") key of the bytes it covers: the logical block, or its disk frame zero-padded
    to PSIZE.  Re-stamped."""
    s = np.array(stream, dtype=np.uint8, copy=True)
    hf, ct = (sha256_key, SHA256) if name == "sha256" else (sha512_key, SHA512)
    for off, po, pl, t in records(s):
        if t != 3 or s[off + 50] != 0 or s[off + 48] != FLETCHER4:
            continue
        lsize, psize, dc, _ = unprop(get_key(s, off)[2])
        logical = s[po:po + pl]
        if dc in (DC_LZ4, DC_LZJB, DC_ZLE):
            fr = disk_frame(oracle, logical, 9, dc).tobytes()
            data = fr[:psize] + bytes(max(0, psize - len(fr)))
        else:
            data = logical.tobytes()
        set_key(s, off, ct, hf(data))
    assert oracle.stream_restamp(s)[0] == 0
    return s


def block_check_lzjb(oracle, inp, mode=VERIFY, frames=False, lzjb=True, sha256=False, sha512=False, out=None):
    """The counters of the block check in `mode` (VERIFY, or RECOMPRESS with its output `out`) with MTZ_FLAG_BLOCK_FRAMES = `frames` and MTZ_FLAG_BLOCK_LZJB =
    `lzjb`: block_frames_ref's model (block_check_frames with `frames`, else block_check) with every
    still-skipped record whose checkable key covers an lzjb or zle frame compared -- as it arrives when
    it arrives as that frame, against encoder_frame() when it arrives raw in VERIFY.
    counters["lzjb_encoded"] / ["zle_encoded"] count the frames encoded."""
    if mode == VERIFY and frames:
        verdicts, st = _F.block_check_frames(oracle, inp, sha256=sha256, sha512=sha512)
    else:
        verdicts, st = _F.block_check(inp, out, mode, sha256=sha256, sha512=sha512)
        st["frames_encoded"] = 0
    st["lzjb_encoded"] = st["zle_encoded"] = 0
    if not lzjb:
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
        if ctype not in hashes or p == 0 or crypt or lsize != drr_lsize or dc not in (DC_LZJB, DC_ZLE):
            continue
        if arrive == dc and mode in (VERIFY, RECOMPRESS):
            fr = b[po:po + pl]
        elif arrive == 0 and mode == VERIFY:
            fr = encoder_frame(dc, b[po:po + pl])
            st["lzjb_encoded" if dc == DC_LZJB else "zle_encoded"] += 1
        else:
            continue
        ok = fr is not None and len(fr) <= psize and hashes[ctype](fr + bytes(psize - len(fr))) == key
        verdicts[i] = FRAME_OK if ok else FRAME_MISS
        st["skipped"] -= 1
        st["frame_ok" if ok else "frame_miss"] += 1
        if not ok:
            st["first_frame_miss"] = min(st["first_frame_miss"], i)
        if ctype in (SHA256, SHA512):
            st["sha256" if ctype == SHA256 else "sha512"] += 1
    return verdicts, st
