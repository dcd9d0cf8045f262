"""The high-ratio LZ4 encoder of MTZ_FLAG_LZ4_HC on the CPU (test infrastructure): ctypes over
tests/lz4hc_ref.c.

The stream walk is oracle/stream.c's own, compiled a second time with the HC frame encoder in place of
orc_zfs_lz4_compress, so `stream_compress(s, hc=True)` differs from `oracle.stream_compress(s)` only in
the encoder of the DRR_WRITE payloads.  Compiled once into a temporary directory keyed by the sources'
hash (the tree may be read-only)."""
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORC = os.path.join(os.path.dirname(_HERE), "oracle")
_SRCS = [os.path.join(_HERE, "lz4hc_ref.c")] + [os.path.join(_ORC, f) for f in
                                                  ("stream.c", "fletcher4.c", "lz4_zfs.c", "mtz_oracle.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        import oracle
        key = hashlib.sha256(b"".join(open(s, "rb").read() for s in _SRCS)).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "mtz_lz4hc_oracle_%d" % os.getuid())
        so = os.path.join(d, "lz4hc_%s.so" % key)
        if not os.path.exists(so):
            os.makedirs(d, exist_ok=True)
            tmp = tempfile.mkdtemp(dir=d)
            cc = [os.environ.get("CC", "gcc"), "-O2", "-std=gnu11", "-Wall", "-fPIC", "-I", _ORC]
            objs = []
            for src, defs in ((_SRCS[0], []), (_SRCS[2], []), (_SRCS[3], []),
                              (_SRCS[1], ["-Dorc_zfs_lz4_compress=orc_zfs_lz4hc_compress",
                                          "-Dorc_stream_compress=orc_stream_compress_hc"])):
                o = os.path.join(tmp, os.path.basename(src) + ".o")
                subprocess.check_call(cc + defs + ["-c", "-o", o, src])
                objs.append(o)
            out = os.path.join(tmp, "lib.so")
            subprocess.check_call(cc + ["-shared", "-o", out] + objs)
            os.replace(out, so)
            shutil.rmtree(tmp, ignore_errors=True)
        L = C.CDLL(so)
        vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
        L.orc_lz4hc_compress_block.argtypes = [vp, i32, vp, i32]
        L.orc_lz4hc_compress_block.restype = i32
        L.orc_zfs_lz4hc_compress.argtypes = [vp, sz, vp]
        L.orc_zfs_lz4hc_compress.restype = sz
        L.orc_stream_compress_hc.argtypes = [vp, sz, vp, sz, C.POINTER(sz), C.POINTER(oracle.StreamStats)]
        L.orc_stream_compress_hc.restype = i32
        _lib = L
    return _lib


def _u8(buf):
    if isinstance(buf, np.ndarray):
        return np.ascontiguousarray(buf.view(np.uint8))
    return np.frombuffer(bytes(buf), dtype=np.uint8)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def lz4hc_compress_block(src, cap=None):
    """the raw LZ4 block (numpy uint8), or None when it does not fit in `cap` bytes"""
    a = _u8(src)
    cap = a.size + a.size // 255 + 64 if cap is None else cap
    dst = np.zeros(cap + 1, dtype=np.uint8)
    n = lib().orc_lz4hc_compress_block(_p(a), a.size, _p(dst), cap)
    return dst[:n].copy() if n > 0 else None


def zfs_lz4hc_compress(src):
    """(psize, frame padded to psize), or (lsize, None) when the block is stored raw"""
    a = _u8(src)
    dst = np.zeros(a.size + 1024, dtype=np.uint8)
    ps = lib().orc_zfs_lz4hc_compress(_p(a), a.size, _p(dst))
    return ps, (dst[:ps].copy() if ps < a.size else None)


def stream_compress(stream, hc=True, cap=None):
    """COMPRESS of a send stream as oracle.stream_compress returns it: (rc, output, stats); with hc the
    DRR_WRITE payloads are this encoder's frames"""
    import oracle
    if not hc:
        return oracle.stream_compress(stream, cap)
    a = _u8(stream)
    cap = a.size * 2 + (1 << 20) if cap is None else cap
    out = np.empty(cap, dtype=np.uint8)
    n = C.c_size_t(0)
    st = oracle.StreamStats()
    rc = lib().orc_stream_compress_hc(_p(a), a.size, _p(out), out.size, C.byref(n), C.byref(st))
    return rc, out[:n.value], st
