"""Reference model of MTZ_FLAG_GZIP_WIRE: gzip frames on the compressed wire.  Test infrastructure, built on
compressed_in_ref and gzip_in_ref.

  expected(x)  COMPRESS with MTZ_FLAG_COMPRESSED_IN | MTZ_FLAG_GZIP_WIRE of the `zfs send -c` stream x:
               COMPRESS of plain(x) with every record that arrived LZ4 or gzip-1 .. gzip-9 put back as it
               arrived, re-stamped, and WIRE_F_GZIP set in every preamble.
  plain(x)     DECOMPRESS with MTZ_FLAG_GZIP_WIRE of that wire: gzip_in_ref.plain(x), the stream `zfs
               send` without -c would have produced.
  verdict(x)   (None, counters) or (index of the failing record, counters) of that COMPRESS.

The wire size follows: every forwarded record costs exactly what it cost in x, so a stream whose every
DRR_WRITE arrives LZ4 or gzip is as long on the wire as x plus one 32-byte preamble per BEGIN."""
import struct

import numpy as np

import block_ref as B
import compressed_in_ref as M
import gzip_in_ref as G

GZIP_WIRE = 2048            # MTZ_FLAG_GZIP_WIRE
WIRE_F_GZIP = 2
PRE_BYTES = 32

plain = G.plain


def forwarded(comp):
    """the compressions COMPRESS with the flag forwards as they arrive"""
    return comp == M.DC_LZ4 or G.is_gzip(comp)


def preambles(oracle, wire):
    """offsets of the wire preambles in `wire`"""
    w = np.asarray(wire, dtype=np.uint8)
    m = np.frombuffer(oracle.WIRE_MAGIC, dtype=np.uint8)
    at = np.flatnonzero(w[:max(w.size - 7, 0)] == m[0])
    for k in range(1, m.size):
        at = at[w[at + k] == m[k]]
    return [int(i) for i in at]


def pre_flags(oracle, wire):
    """the capability bits of each preamble of `wire`"""
    w = np.asarray(wire, dtype=np.uint8).tobytes()
    return [struct.unpack_from("<I", w, i + 12)[0] for i in preambles(oracle, wire)]


def set_pre_flags(oracle, wire, on=0, off=0):
    """`wire` with bits `on` set and `off` cleared in every preamble (outside the stream checksum)"""
    w = np.array(wire, dtype=np.uint8, copy=True)
    for i in preambles(oracle, w):
        f = (struct.unpack("<I", w[i + 12:i + 16].tobytes())[0] | on) & ~off
        w[i + 12:i + 16] = np.frombuffer(struct.pack("<I", f), dtype=np.uint8)
    return w


def splice(oracle, wire, x):
    """`wire` (a COMPRESS output of plain(x), preambles included) with every record of x that arrived LZ4
    or gzip put back as it arrived, re-stamped, and WIRE_F_GZIP set in each preamble"""
    w = np.asarray(wire, dtype=np.uint8)
    body = oracle.wire_strip(w)
    pres = [w[i:i + PRE_BYTES].copy() for i in preambles(oracle, w)]
    xb = np.asarray(x, dtype=np.uint8)
    xr, wr = B.records(xb), B.records(body)
    assert len(xr) == len(wr)
    parts, k = [], 0
    for (xo, xpo, xpl, t), (wo, wpo, wpl, _) in zip(xr, wr):
        if t == 0:
            parts.append(pres[k])
            k += 1
        if t == 3 and forwarded(int(xb[xo + 50])):
            parts.append(xb[xo:xpo + xpl])
        else:
            parts.append(body[wo:wpo + wpl])
    out = np.ascontiguousarray(np.concatenate(parts))
    pos = preambles(oracle, out) + [out.size]
    for a, e in zip(pos, pos[1:]):
        seg = np.ascontiguousarray(out[a + PRE_BYTES:e])
        assert oracle.stream_restamp(seg)[0] == 0
        out[a + PRE_BYTES:e] = seg
    return set_pre_flags(oracle, out, on=WIRE_F_GZIP)


def expected(oracle, x):
    """COMPRESS with MTZ_FLAG_COMPRESSED_IN | MTZ_FLAG_GZIP_WIRE of x (a stream the stage accepts), with
    ZFS's LZ4 encoder"""
    rc, w, _ = oracle.stream_compress(plain(oracle, x))
    assert rc == 0
    return splice(oracle, w, x)


def verdict(oracle, x):
    """(first failing record or None, the counters of mtz_compressed_in_stats of that COMPRESS)"""
    st = {"lz4_passed": 0, "lzjb_decoded": 0, "zle_decoded": 0, "gzip_decoded": 0, "gzip_passed": 0}
    b = np.asarray(x, dtype=np.uint8)
    for i, (off, po, pl, t) in enumerate(B.records(b)):
        if t != 3 or b[off + 50] == 0:
            continue
        c = int(b[off + 50])
        if forwarded(c):
            st["gzip_passed" if G.is_gzip(c) else "lz4_passed"] += 1
            continue
        if M.decode(oracle, c, b[po:po + pl], M._lsize(b[off:off + 312])) is None:
            return i, st
        st["lzjb_decoded" if c == M.DC_LZJB else "zle_decoded"] += 1
    return None, st


def receiver_verdict(oracle, wire):
    """(first failing record or None, mtz_compressed_in_stats) of DECOMPRESS with the flag over `wire`:
    gzip records are inflated by gzip_in_ref's rule; nothing else is counted there"""
    st = {"lz4_passed": 0, "lzjb_decoded": 0, "zle_decoded": 0, "gzip_decoded": 0, "gzip_passed": 0}
    b = oracle.wire_strip(np.asarray(wire, dtype=np.uint8))
    for i, (off, po, pl, t) in enumerate(B.records(b)):
        if t != 3 or not G.is_gzip(int(b[off + 50])):
            continue
        if G.inflate(b[po:po + pl], M._lsize(b[off:off + 312])) is None:
            return i, st
        st["gzip_decoded"] += 1
    return None, st


def wire_size(oracle, x):
    """len(expected(x)) without running an encoder, for a stream whose every DRR_WRITE arrives LZ4 or
    gzip: the send -c size plus one preamble per BEGIN"""
    b = np.asarray(x, dtype=np.uint8)
    recs = B.records(b)
    assert all(t != 3 or forwarded(int(b[off + 50])) for off, _, _, t in recs)
    return b.size + PRE_BYTES * sum(1 for _, _, _, t in recs if t == 0)
