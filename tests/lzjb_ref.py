"""The lzjb / zle encoders and decoders of ZFS, restated twice.  Test infrastructure: plain Python,
numpy, ctypes and tests/lzjb_zfs.c.

tests/lzjb_zfs.c is ZFS's C code on real pointers (`phase` = the source buffer's address mod 1024, which
lzjb's output depends on), compiled on first use; py_lzjb_compress and py_zle_compress are an
independent pure-Python restatement that models phase 0 the way the GPU does: a table entry is the
position's low 16 bits, 0 for "never written"."""
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

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
